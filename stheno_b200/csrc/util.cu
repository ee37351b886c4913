// K4 and layout helpers: log-marginal finish, row reductions, padding / symmetrisation / transposition,
// the DMMA peak probe and the launch counter.
#include <math.h>

#include "common.cuh"

namespace gpk {

long long g_launch_count = 0;

// ---- logpdf finish: out[b][c] = -0.5 (logdet[b] + n log 2pi + sum_j a[b][c][j]^2) -------------------------------
// stheno/random.py:272-279.  One CTA per (c, b); a HBM-read-bound row reduction.  fp64 sums in both precisions: in fp32,
// each thread adds n_cols / 512 terms in sequence, and a running sum near 1 would drop every term below 2^-25.
template <typename T>
__global__ void logpdf_finish_kernel(const T* __restrict__ a, int64_t lda, int64_t a_bs, int64_t n, int64_t n_cols,
                                     int32_t k, const T* __restrict__ logdet, T* __restrict__ out) {
  const int c = blockIdx.x, b = blockIdx.y;
  const T* row = a + (int64_t)b * a_bs + (int64_t)c * lda;
  double s = 0.0;
  for (int64_t j = threadIdx.x; j < n_cols; j += blockDim.x) {
    const double v = (double)row[j];
    s = fma(v, v, s);
  }
  __shared__ double red[32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    const double log2pi = 1.8378770664093454835606594728112;
    out[(int64_t)b * k + c] = (T)(-((double)logdet[b] + (double)n * log2pi + t) / 2.0);
  }
}

// ---- row reductions: dot[r] = <V[r,:], b>, sq[r] = |V[r,:]|^2 ; one warp per row, fp64 sums in both precisions ---------
template <typename T>
__global__ void row_dot_sq_kernel(const T* __restrict__ V, int64_t ldv, int64_t v_bs, int64_t rows, int64_t n_cols,
                                  const T* __restrict__ bvec, int64_t b_bs, T* __restrict__ dot, T* __restrict__ sq,
                                  int64_t o_bs) {
  const int bidx = blockIdx.y;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const T* row = V + (int64_t)bidx * v_bs + r * ldv;
  const T* bv = bvec ? bvec + (int64_t)bidx * b_bs : nullptr;
  double sd = 0.0, ss = 0.0;
  for (int64_t j = lane; j < n_cols; j += 32) {
    const double v = (double)row[j];
    ss = fma(v, v, ss);
    if (bv) sd = fma(v, (double)bv[j], sd);
  }
  sd = warp_sum(sd);
  ss = warp_sum(ss);
  if (lane == 0) {
    if (dot) dot[(int64_t)bidx * o_bs + r] = (T)sd;
    if (sq) sq[(int64_t)bidx * o_bs + r] = (T)ss;
  }
}

// ---- pad copy --------------------------------------------------------------------------------------------------
template <typename T>
__global__ void pad_copy_kernel(const T* __restrict__ src, int64_t lds, int64_t s_bs, int64_t rows, int64_t cols,
                                T* __restrict__ dst, int64_t ldd, int64_t d_bs, int64_t rows_pad, int64_t cols_pad,
                                T diag_add, int32_t pad_identity) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.z;
  if (c >= cols_pad) return;
  for (int64_t r = blockIdx.y; r < rows_pad; r += gridDim.y) {  // grid.y is capped at 65535
    T v;
    if (r < rows && c < cols) {
      v = src[(int64_t)b * s_bs + r * lds + c];
      if (r == c) v += diag_add;
    } else {
      v = (pad_identity && r == c) ? T(1) : T(0);
    }
    dst[(int64_t)b * d_bs + r * ldd + c] = v;
  }
}

// mirror lower -> upper, 32 x 32 tiles through shared memory
template <typename T>
__global__ void symmetrize_kernel(T* __restrict__ A, int64_t lda, int64_t a_bs, int64_t n) {
  __shared__ T tile[32][33];
  const int tr = blockIdx.y, tc = blockIdx.x;
  if (tc > tr) return;
  A += (int64_t)blockIdx.z * a_bs;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int64_t r = (int64_t)tr * 32 + i, c = (int64_t)tc * 32 + tx;
    tile[i][tx] = (r < n && c < n) ? A[r * lda + c] : T(0);
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    // destination element (row = tc*32 + i, col = tr*32 + tx) = source (tr*32 + tx, tc*32 + i)
    const int64_t r = (int64_t)tc * 32 + i, c = (int64_t)tr * 32 + tx;
    if (r < n && c < n && c > r) A[r * lda + c] = tile[tx][i];
  }
}

template <typename T>
__global__ void transpose_kernel(const T* __restrict__ src, int64_t lds, int64_t s_bs, int64_t rows, int64_t cols,
                                 T* __restrict__ dst, int64_t ldd, int64_t d_bs) {
  __shared__ T tile[32][33];
  src += (int64_t)blockIdx.z * s_bs;
  dst += (int64_t)blockIdx.z * d_bs;
  const int tx = threadIdx.x, ty = threadIdx.y;
  // row tiles on grid.x (no 65535 limit: rows may be a whole data set); column tiles strided over grid.y
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  for (int64_t c0 = (int64_t)blockIdx.y * 32; c0 < cols; c0 += (int64_t)gridDim.y * 32) {
    for (int i = ty; i < 32; i += 8) {
      const int64_t r = r0 + i, c = c0 + tx;
      tile[i][tx] = (r < rows && c < cols) ? src[r * lds + c] : T(0);
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
      const int64_t r = c0 + i, c = r0 + tx;  // dst is cols x rows
      if (r < cols && c < rows) dst[r * ldd + c] = tile[tx][i];
    }
    __syncthreads();
  }
}

// ---- DMMA peak probe --------------------------------------------------------------------------------------------
__global__ void dmma_probe_kernel(double* out, int iters, double a, double b) {
  double c[8][2];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    c[i][0] = threadIdx.x;
    c[i][1] = i;
  }
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) dmma884(c[i][0], c[i][1], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int row_dot_sq(const double* V, int64_t ldv, int64_t rows, int64_t n_cols, const double* b, double* dot, double* sq,
               cudaStream_t stream) {
  return gpk_row_dot_sq_f64(V, ldv, 0, rows, n_cols, b, 0, dot, sq, 0, 1, stream);
}
int row_dot_sq(const float* V, int64_t ldv, int64_t rows, int64_t n_cols, const float* b, float* dot, float* sq,
               cudaStream_t stream) {
  return gpk_row_dot_sq_f32(V, ldv, 0, rows, n_cols, b, 0, dot, sq, 0, 1, stream);
}

}  // namespace gpk

#define GPK_DEFINE_UTILS(SUF, T)                                                                                       \
  int gpk_logpdf_finish_##SUF(const T* a, int64_t lda, int64_t a_bstride, int64_t n, int64_t n_cols, int32_t k,        \
                              const T* logdet, T* out, int32_t batch, void* stream) {                                  \
    if (!a || !logdet || !out || k < 1 || batch < 1 || n_cols < 0) return GPK_ERR_ARG;                                 \
    dim3 grid((unsigned)k, (unsigned)batch);                                                                           \
    gpk::logpdf_finish_kernel<T><<<grid, 512, 0, (cudaStream_t)stream>>>(a, lda, a_bstride, n, n_cols, k, logdet, out); \
    GPK_COUNT_LAUNCH();                                                                                                \
    GPK_CHECK_LAUNCH();                                                                                                \
    return 0;                                                                                                          \
  }                                                                                                                    \
  int gpk_row_dot_sq_##SUF(const T* V, int64_t ldv, int64_t v_bstride, int64_t rows, int64_t n_cols, const T* b,       \
                           int64_t b_bstride, T* dot, T* sq, int64_t o_bstride, int32_t batch, void* stream) {         \
    if (!V || rows < 0 || n_cols < 0 || batch < 1) return GPK_ERR_ARG;                                                 \
    if (rows == 0) return 0;                                                                                           \
    dim3 grid((unsigned)((rows + 7) / 8), (unsigned)batch);                                                            \
    gpk::row_dot_sq_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>(V, ldv, v_bstride, rows, n_cols, b, b_bstride,   \
                                                                     dot, sq, o_bstride);                              \
    GPK_COUNT_LAUNCH();                                                                                                \
    GPK_CHECK_LAUNCH();                                                                                                \
    return 0;                                                                                                          \
  }                                                                                                                    \
  int gpk_pad_copy_##SUF(const T* src, int64_t lds, int64_t s_bstride, int64_t rows, int64_t cols, T* dst,             \
                         int64_t ldd, int64_t d_bstride, int64_t rows_pad, int64_t cols_pad, double diag_add,          \
                         int32_t pad_identity, int32_t batch, void* stream) {                                          \
    if (!dst || rows < 0 || cols < 0 || rows_pad < rows || cols_pad < cols || batch < 1) return GPK_ERR_ARG;           \
    if (rows_pad == 0 || cols_pad == 0) return 0;                                                                      \
    dim3 grid((unsigned)((cols_pad + 255) / 256), (unsigned)(rows_pad < 65535 ? rows_pad : 65535), (unsigned)batch);   \
    gpk::pad_copy_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>(src, lds, s_bstride, rows, cols, dst, ldd,         \
                                                                   d_bstride, rows_pad, cols_pad, (T)diag_add,         \
                                                                   pad_identity);                                      \
    GPK_COUNT_LAUNCH();                                                                                                \
    GPK_CHECK_LAUNCH();                                                                                                \
    return 0;                                                                                                          \
  }                                                                                                                    \
  int gpk_symmetrize_##SUF(T* A, int64_t lda, int64_t a_bstride, int64_t n, int32_t batch, void* stream) {             \
    if (!A || n < 0 || batch < 1) return GPK_ERR_ARG;                                                                  \
    if (n == 0) return 0;                                                                                              \
    const unsigned t = (unsigned)((n + 31) / 32);                                                                      \
    dim3 grid(t, t, (unsigned)batch), block(32, 8);                                                                    \
    gpk::symmetrize_kernel<T><<<grid, block, 0, (cudaStream_t)stream>>>(A, lda, a_bstride, n);                         \
    GPK_COUNT_LAUNCH();                                                                                                \
    GPK_CHECK_LAUNCH();                                                                                                \
    return 0;                                                                                                          \
  }                                                                                                                    \
  int gpk_transpose_##SUF(const T* src, int64_t lds, int64_t s_bstride, int64_t rows, int64_t cols, T* dst,            \
                          int64_t ldd, int64_t d_bstride, int32_t batch, void* stream) {                               \
    if (!src || !dst || rows < 0 || cols < 0 || batch < 1) return GPK_ERR_ARG;                                         \
    if (rows == 0 || cols == 0) return 0;                                                                              \
    const int64_t col_tiles = (cols + 31) / 32;                                                                        \
    dim3 grid((unsigned)((rows + 31) / 32), (unsigned)(col_tiles < 65535 ? col_tiles : 65535), (unsigned)batch),       \
        block(32, 8);                                                                                                  \
    gpk::transpose_kernel<T><<<grid, block, 0, (cudaStream_t)stream>>>(src, lds, s_bstride, rows, cols, dst, ldd,      \
                                                                      d_bstride);                                      \
    GPK_COUNT_LAUNCH();                                                                                                \
    GPK_CHECK_LAUNCH();                                                                                                \
    return 0;                                                                                                          \
  }

extern "C" {

GPK_DEFINE_UTILS(f64, double)
GPK_DEFINE_UTILS(f32, float)

int gpk_version(void) { return GPK_VERSION; }
int64_t gpk_round_up(int64_t n) { return (n + GPK_TILE - 1) / GPK_TILE * GPK_TILE; }
int64_t gpk_launch_count(void) { return gpk::g_launch_count; }
void gpk_launch_count_reset(void) { gpk::g_launch_count = 0; }

double gpk_probe_dmma_tflops(void) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1.0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1.0;
  double* out = nullptr;
  const int threads = 256, iters = 20000;
  if (cudaMalloc(&out, sizeof(double) * sms * threads) != cudaSuccess) return -2.0;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  gpk::dmma_probe_kernel<<<sms, threads>>>(out, iters, 1.0000001, 0.9999999);
  cudaDeviceSynchronize();
  float best = 1e30f;
  for (int rep = 0; rep < 3; ++rep) {
    cudaEventRecord(e0);
    gpk::dmma_probe_kernel<<<sms, threads>>>(out, iters, 1.0000001, 0.9999999);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    if (ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(out);
  if (cudaGetLastError() != cudaSuccess) return -3.0;
  // 8 DMMA.8x8x4 per iteration per warp, 512 flop each
  return 512.0 * 8 * iters * (threads / 32) * sms / (best * 1e-3) / 1e12;
}
}
