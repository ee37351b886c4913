// K1: fused pairwise-distance + kernel-evaluation kernel (sm_90a).
//
// One CTA produces a 64 x 64 tile of K.  The pre-stretched input rows of the tile (x^(g) and y^(g) for every
// lengthscale group g) are staged into shared memory by the TMA engine with 1-D bulk async copies
// (cp.async.bulk + mbarrier; SASS UBLKCP), falling back to plain loads for unaligned / ragged tiles.  Every
// thread owns a 4 x 4 micro-tile (columns strided by 16 so that a half-warp reads conflict-free shared memory
// and writes one contiguous 128-byte (fp64) row segment per store), evaluates the flattened sum-of-products kernel
// expression in registers and writes K exactly once, with the observation noise, the Cholesky jitter and the
// identity padding fused in.  In LOWER mode tiles above the diagonal are skipped (halves the exp work and the
// HBM writes).  Roofline: HBM-write bound (8 n^2 bytes, 4 n^2 in LOWER mode), close to the fp64-ALU ridge.
//
// Reference arithmetic replaced: mlkernels.pairwise for EQ/Matern/Linear/Delta and Scaled/Sum/Product/Stretched
// (call sites stheno/model/fdd.py:79, stheno/model/observations.py:139,285,286), Dense + Diagonal (fdd.py:79)
// and B.reg's "+ epsilon I" (README.md:820-830).
#include "common.cuh"

namespace gpk {

constexpr int KM_TILE = 64;
constexpr int KM_THREADS = 256;

struct KmParams {
  gpk_kernel_desc desc;
  const void* xg;
  const void* yg;
  int64_t xg_gstride, x_bstride, yg_gstride, y_bstride;
  int64_t n, n2;
  int32_t d;
  double noise_scalar;
  const void* noise_vec;
  int64_t nv_bstride;
  double jitter;
  int32_t flags;
  void* out;
  int64_t ldo, o_bstride;
  int64_t rows_out, cols_out;
};

// phi(kind) from squared distance d2 / dot product.  d == 1 mirrors lab's |x - y| special case (no 1e-30 clamp).
template <typename T>
__device__ __forceinline__ T eval_factor(int kind, T d2, T dot, bool same_point, bool same_obj, int d, double param = 0.0) {
  switch (kind) {
    case GPK_RQ: {  // (1 + r^2 / (2 alpha))^-alpha
      const double a = param;
      return (T)exp(-a * log1p((double)d2 / (2.0 * a)));
    }
    case GPK_EQ:
      return t_exp<T>(T(-0.5) * d2);
    case GPK_MATERN12: {
      T r = (d == 1) ? t_sqrt<T>(d2) : t_sqrt<T>(d2 > T(1e-30) ? d2 : T(1e-30));
      return t_exp<T>(-r);
    }
    case GPK_MATERN32: {
      T r = (d == 1) ? t_sqrt<T>(d2) : t_sqrt<T>(d2 > T(1e-30) ? d2 : T(1e-30));
      T s = T(1.7320508075688772) * r;
      return (T(1) + s) * t_exp<T>(-s);
    }
    case GPK_MATERN52: {
      T r = (d == 1) ? t_sqrt<T>(d2) : t_sqrt<T>(d2 > T(1e-30) ? d2 : T(1e-30));
      T s = T(2.23606797749979) * r;
      return (T(1) + s + T(1.6666666666666667) * d2) * t_exp<T>(-s);
    }
    case GPK_LINEAR:
      return dot;
    case GPK_DELTA:
      return same_obj ? (same_point ? T(1) : T(0)) : (d2 < T(1e-10) ? T(1) : T(0));
    default:
      return T(1);
  }
}

template <typename T>
__global__ void __launch_bounds__(KM_THREADS) kernel_matrix_kernel(const KmParams p) {
  const int tile_c = blockIdx.x, tile_r = blockIdx.y, b = blockIdx.z;
  const bool lower = p.flags & GPK_KM_LOWER;
  // LOWER: skip tiles strictly above the diagonal at 128-granularity (the Cholesky's tile size), so that every
  // 128 x 128 diagonal tile is fully initialised.
  if (lower && (tile_c >> 1) > (tile_r >> 1)) return;
  const bool same_obj = p.flags & GPK_KM_SAME;
  const int d = p.d;
  const int G = p.desc.n_groups;
  const int64_t r0 = (int64_t)tile_r * KM_TILE, c0 = (int64_t)tile_c * KM_TILE;

  extern __shared__ __align__(16) unsigned char km_smem[];
  __shared__ __align__(8) uint64_t bar;
  T* xs = reinterpret_cast<T*>(km_smem);            // [G][64][d]
  T* ys = xs + (size_t)G * KM_TILE * d;               // [G][64][d]
  const T* xg = static_cast<const T*>(p.xg) + (int64_t)b * p.x_bstride;
  const T* yg = static_cast<const T*>(p.yg) + (int64_t)b * p.y_bstride;

  // rows of the tile that exist in the inputs (the rest is padding)
  const int xr = (int)max((int64_t)0, min((int64_t)KM_TILE, p.n - r0));
  const int yr = (int)max((int64_t)0, min((int64_t)KM_TILE, p.n2 - c0));
  const uint32_t xbytes = (uint32_t)xr * d * sizeof(T), ybytes = (uint32_t)yr * d * sizeof(T);
  // The bulk-copy engine needs 16-byte aligned addresses and sizes.
  bool bulk = (xbytes % 16 == 0) && (ybytes % 16 == 0) && ((KM_TILE * d * sizeof(T)) % 16 == 0);
  for (int g = 0; g < G && bulk; ++g) {
    bulk = bulk && (reinterpret_cast<uintptr_t>(xg + g * p.xg_gstride + r0 * d) % 16 == 0) &&
           (reinterpret_cast<uintptr_t>(yg + g * p.yg_gstride + c0 * d) % 16 == 0);
  }
  if (bulk) {
    if (threadIdx.x == 0) {
      mbar_init(&bar, 1);
      fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(&bar, (uint32_t)G * (xbytes + ybytes));
      for (int g = 0; g < G; ++g) {
        if (xbytes) bulk_copy_g2s(xs + (size_t)g * KM_TILE * d, xg + g * p.xg_gstride + r0 * d, xbytes, &bar);
        if (ybytes) bulk_copy_g2s(ys + (size_t)g * KM_TILE * d, yg + g * p.yg_gstride + c0 * d, ybytes, &bar);
      }
    }
    mbar_wait(&bar, 0);
  } else {
    for (int g = 0; g < G; ++g) {
      for (int i = threadIdx.x; i < xr * d; i += KM_THREADS)
        xs[(size_t)g * KM_TILE * d + i] = xg[g * p.xg_gstride + r0 * d + i];
      for (int i = threadIdx.x; i < yr * d; i += KM_THREADS)
        ys[(size_t)g * KM_TILE * d + i] = yg[g * p.yg_gstride + c0 * d + i];
    }
    __syncthreads();
  }

  // Transpose the y rows to [g][k][64 (+1 pad)] so that the 16 column-threads of a half-warp read consecutive
  // shared-memory words (the [row][d] image the bulk copy produces would be a d-word stride: bank conflicts).
  T* yt = ys + (size_t)G * KM_TILE * d;  // [G][d][65]
  for (int idx = threadIdx.x; idx < G * KM_TILE * d; idx += KM_THREADS) {
    const int g = idx / (KM_TILE * d), rem = idx - g * KM_TILE * d;
    const int c = rem / d, k = rem - c * d;
    yt[((size_t)g * d + k) * (KM_TILE + 1) + c] = ys[idx];
  }
  __syncthreads();

  // thread (tx, ty): rows r0 + 4*ty + i, columns c0 + tx + 16*j  (i, j < 4)
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  T acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = T(0);

  T d2[4][4], dt[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      d2[i][j] = T(0);
      dt[i][j] = T(0);
    }
  int last_g = -1;
  for (int t = 0; t < p.desc.n_terms; ++t) {
    T prod[4][4];
    const T coef = (T)p.desc.coef[t];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) prod[i][j] = coef;
    for (int f = p.desc.term_begin[t]; f < p.desc.term_begin[t + 1]; ++f) {
      const int kind = p.desc.fac_kind[f];
      const int g = p.desc.fac_group[f];
      if ((g != last_g || kind == GPK_LINEAR) && kind != GPK_ONE && !(kind == GPK_DELTA && same_obj)) {
        last_g = g;
        const T* xr_ = xs + ((size_t)g * KM_TILE + ty * 4) * d;
        const T* yc_ = yt + (size_t)g * d * (KM_TILE + 1) + tx;
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            d2[i][j] = T(0);
            dt[i][j] = T(0);
          }
        if (kind == GPK_LINEAR) {  // inner products only for the Linear kernel (warp-uniform branch)
          for (int k = 0; k < d; ++k) {
            T xv[4], yv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) xv[i] = xr_[i * d + k];
#pragma unroll
            for (int j = 0; j < 4; ++j) yv[j] = yc_[(size_t)k * (KM_TILE + 1) + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int j = 0; j < 4; ++j) dt[i][j] = fma(xv[i], yv[j], dt[i][j]);
          }
          last_g = -1;  // d2 was not formed: a following distance-based factor of the same group recomputes
        } else {
#pragma unroll 2
          for (int k = 0; k < d; ++k) {
            T xv[4], yv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) xv[i] = xr_[i * d + k];
#pragma unroll
            for (int j = 0; j < 4; ++j) yv[j] = yc_[(size_t)k * (KM_TILE + 1) + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                T df = xv[i] - yv[j];
                d2[i][j] = fma(df, df, d2[i][j]);
              }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool same_pt = (r0 + ty * 4 + i) == (c0 + tx + 16 * j);
          prod[i][j] *= eval_factor<T>(kind, d2[i][j], dt[i][j], same_pt, same_obj, d, p.desc.fac_param[f]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] += prod[i][j];
  }

  // epilogue: diagonal terms, identity / zero padding; a half-warp writes 128 (fp64) / 64 (fp32) contiguous bytes
  T* out = static_cast<T*>(p.out) + (int64_t)b * p.o_bstride;
  const T* nv = p.noise_vec ? static_cast<const T*>(p.noise_vec) + (int64_t)b * p.nv_bstride : nullptr;
  const bool pad_id = p.flags & GPK_KM_PAD_IDENTITY;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t r = r0 + ty * 4 + i;
    if (r >= p.rows_out) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t c = c0 + tx + 16 * j;
      if (c >= p.cols_out) continue;
      T val = acc[i][j];
      if (r >= p.n || c >= p.n2) {
        val = (pad_id && r == c) ? T(1) : T(0);
      } else if (same_obj && r == c) {
        val += (T)p.noise_scalar;
        if (nv) val += nv[r];
        val += (T)p.jitter;
      }
      out[r * p.ldo + c] = val;
    }
  }
}

// ---- fast path: ONE stationary factor (coef * EQ / Matern12 / 32 / 52 of one length-scale group) ------------------------
// The benchmarked configurations all reduce to this (the Delta / noise part is a diagonal term of the epilogue).  Against the
// generic kernel above (ncu r02: FP64 pipe 20 % busy, 165 registers -> one CTA of 8 warps per SM, issue slots mostly idle):
//   * the factor kind is a template parameter: no per-element switch, d2 is the only 16-element array kept in registers
//     (<= 128 registers, >= 2 CTAs per SM so one CTA's TMA wait / transpose / barrier hides under the other's arithmetic);
//   * fp64 exp = 2^(k/64) table (shared memory) x degree-5 polynomial on |r| <= ln2/128 with a two-part Cody-Waite reduction:
//     11 FP64-pipe operations instead of the ~25 of the library exp (which also handles overflow / NaN paths that a
//     non-positive argument never takes); relative error <= 4.0e-16 (at most 2 ulp; table entry rounding + 5 Horner
//     steps), i.e. well inside the 1e-12 parity budget on K (tests/test_gpu_primitives.py compares at rtol 1e-12 against
//     the oracle).  Results below the normal range (x < -708.4) are flushed to 0 where the library exp returns a denormal.
//     tests/_fexp_model.py restates this function operation for operation; tests/test_kernel_edges.py checks it.
__device__ __forceinline__ double fast_exp_nonpos(double x, const double* __restrict__ tab) {
  // x <= 0.  k = round(x * 64 / ln2); x = k * ln2/64 + r; exp(x) = 2^(k >> 6) * tab[k & 63] * exp(r)
  const double t = fma(x, 92.332482616893656877, 6755399441055744.0);  // 64 / ln2, 1.5 * 2^52: round-to-nearest in the low bits
  const int k = __double2loint(t);
  const double kd = t - 6755399441055744.0;
  double r = fma(kd, -0.010830424696249145, x);    // ln2/64, high part (fma: one rounding, of a result of size <= ln2/128)
  r = fma(kd, -3.623510646634843e-19, r);  // ln2/64 minus the high part
  double p = fma(r, 8.3333333333333332e-3, 4.1666666666666664e-2);
  p = fma(p, r, 1.6666666666666666e-1);
  p = fma(p, r, 0.5);
  p = fma(p, r, 1.0);
  p = fma(p, r, 1.0);
  const double v = p * tab[k & 63];
  const int e = k >> 6;
  // Range check, in the integer pipe: the result is valid for k in [-65408, 0] (k >> 6 >= -1022) with t's high word that
  // of 1.5 * 2^52 + k (0x4337ffff for k < 0, 0x43380000 for k = 0).  Anything else is an exp(x) below the normal range
  // (flushed to 0), -inf, an x so negative that k no longer fits the low 32 bits of t (the exponent arithmetic would write
  // garbage into the sign and exponent bits), or a NaN, which stays a NaN.
  const int ht = __double2hiint(t);
  if ((unsigned)k + 65408u > 65408u || ht - (k >> 31) != 0x43380000) return ((ht & 0x7fffffff) > 0x7ff00000) ? t : 0.0;
  return __hiloint2double(__double2hiint(v) + e * 1048576, __double2loint(v));
}

template <typename T, int KIND>
__device__ __forceinline__ T fast_factor(T d2, int d, const double* tab);
template <>
__device__ __forceinline__ double fast_factor<double, GPK_EQ>(double d2, int, const double* tab) {
  return fast_exp_nonpos(-0.5 * d2, tab);
}
template <>
__device__ __forceinline__ double fast_factor<double, GPK_MATERN12>(double d2, int d, const double* tab) {
  const double r = (d == 1) ? sqrt(d2) : sqrt(d2 > 1e-30 ? d2 : 1e-30);
  return fast_exp_nonpos(-r, tab);
}
template <>
__device__ __forceinline__ double fast_factor<double, GPK_MATERN32>(double d2, int d, const double* tab) {
  const double r = (d == 1) ? sqrt(d2) : sqrt(d2 > 1e-30 ? d2 : 1e-30);
  const double s = 1.7320508075688772 * r;
  return (1.0 + s) * fast_exp_nonpos(-s, tab);
}
template <>
__device__ __forceinline__ double fast_factor<double, GPK_MATERN52>(double d2, int d, const double* tab) {
  const double r = (d == 1) ? sqrt(d2) : sqrt(d2 > 1e-30 ? d2 : 1e-30);
  const double s = 2.23606797749979 * r;
  return (1.0 + s + 1.6666666666666667 * d2) * fast_exp_nonpos(-s, tab);
}
template <>
__device__ __forceinline__ float fast_factor<float, GPK_EQ>(float d2, int, const double*) {
  return expf(-0.5f * d2);
}
template <>
__device__ __forceinline__ float fast_factor<float, GPK_MATERN12>(float d2, int d, const double*) {
  const float r = (d == 1) ? sqrtf(d2) : sqrtf(d2 > 1e-30f ? d2 : 1e-30f);
  return expf(-r);
}
template <>
__device__ __forceinline__ float fast_factor<float, GPK_MATERN32>(float d2, int d, const double*) {
  const float r = (d == 1) ? sqrtf(d2) : sqrtf(d2 > 1e-30f ? d2 : 1e-30f);
  const float s = 1.7320508075688772f * r;
  return (1.0f + s) * expf(-s);
}
template <>
__device__ __forceinline__ float fast_factor<float, GPK_MATERN52>(float d2, int d, const double*) {
  const float r = (d == 1) ? sqrtf(d2) : sqrtf(d2 > 1e-30f ? d2 : 1e-30f);
  const float s = 2.23606797749979f * r;
  return (1.0f + s + 1.6666666666666667f * d2) * expf(-s);
}

constexpr int KM_STRIP = 8;  // column tiles per CTA of the fast kernel

// One CTA = one row tile x a strip of up to KM_STRIP column tiles.  The x rows are staged once; the y rows of tile c + 1 are
// fetched by the TMA engine (double-buffered, one mbarrier per buffer) while tile c is evaluated, so the bulk-copy latency,
// the transposition and the barriers of a tile hide under the arithmetic of its predecessor (round-2 ncu of the
// one-tile-per-CTA version: FP64 pipe 35 % busy with 3 CTAs per SM -- the per-tile prologue was as long as the tile's math).
// n = 16384, lower: 0.499 ms against 0.585 ms for one tile per CTA (1.22 ms for the generic descriptor kernel).
template <typename T, int KIND>
__global__ void __launch_bounds__(KM_THREADS, 3) kernel_matrix_fast_kernel(const KmParams p) {
  const int tile_r = blockIdx.y, b = blockIdx.z;
  const bool lower = p.flags & GPK_KM_LOWER;
  const int tiles_x = (int)((p.cols_out + KM_TILE - 1) / KM_TILE);
  const int c_begin = blockIdx.x * KM_STRIP;
  int c_end = min(c_begin + KM_STRIP, tiles_x);
  // LOWER: tiles strictly above the diagonal at 128-granularity are never written
  if (lower) c_end = min(c_end, ((tile_r >> 1) + 1) * 2);
  if (c_begin >= c_end) return;
  const bool same_obj = p.flags & GPK_KM_SAME;
  const int d = p.d;
  const int g = p.desc.fac_group[0];
  const int64_t r0 = (int64_t)tile_r * KM_TILE;

  extern __shared__ __align__(16) unsigned char km_smem[];
  __shared__ __align__(8) uint64_t bars[2];
  __shared__ double tab[64];
  T* xs = reinterpret_cast<T*>(km_smem);        // [64][d]
  T* ysb = xs + (size_t)KM_TILE * d;             // [2][64][d]
  T* yt = ysb + (size_t)2 * KM_TILE * d;         // [d][65]
  const T* xg = static_cast<const T*>(p.xg) + (int64_t)b * p.x_bstride + g * p.xg_gstride + r0 * d;
  const T* yg0 = static_cast<const T*>(p.yg) + (int64_t)b * p.y_bstride + g * p.yg_gstride;
  if (sizeof(T) == 8 && threadIdx.x < 64) tab[threadIdx.x] = exp2((double)threadIdx.x * 0.015625);

  const int xr = (int)max((int64_t)0, min((int64_t)KM_TILE, p.n - r0));
  const uint32_t xbytes = (uint32_t)xr * d * sizeof(T);
  // the bulk-copy engine needs 16-byte aligned addresses and sizes: every tile of the strip has to qualify
  bool bulk = (xbytes % 16 == 0) && ((KM_TILE * d * sizeof(T)) % 16 == 0) && (reinterpret_cast<uintptr_t>(xg) % 16 == 0) &&
              (reinterpret_cast<uintptr_t>(yg0) % 16 == 0);
  // EVERY tile of the strip has to qualify (16-byte multiple): with identity padding the ragged tile -- the one that contains
  // column n2 -- is followed by empty padding tiles, so looking at the strip's last tile only is not enough (that oversight
  // issued a 24-byte cp.async.bulk whose mbarrier never completed: the hang of the first strip version)
  for (int c = c_begin; c < c_end; ++c) {
    const int yr_c = (int)max((int64_t)0, min((int64_t)KM_TILE, p.n2 - (int64_t)c * KM_TILE));
    bulk = bulk && (((uint32_t)yr_c * d * sizeof(T)) % 16 == 0);
  }
  auto y_rows = [&](int c) { return (int)max((int64_t)0, min((int64_t)KM_TILE, p.n2 - (int64_t)c * KM_TILE)); };
  if (bulk) {
    if (threadIdx.x == 0) {
      mbar_init(&bars[0], 1);
      mbar_init(&bars[1], 1);
      fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {  // x rows + the first y tile arrive on buffer 0's barrier
      const uint32_t yb = (uint32_t)y_rows(c_begin) * d * sizeof(T);
      mbar_arrive_expect_tx(&bars[0], xbytes + yb);
      if (xbytes) bulk_copy_g2s(xs, xg, xbytes, &bars[0]);
      if (yb) bulk_copy_g2s(ysb, yg0 + (int64_t)c_begin * KM_TILE * d, yb, &bars[0]);
    }
  } else {
    for (int i = threadIdx.x; i < xr * d; i += KM_THREADS) xs[i] = xg[i];
  }

  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  T* out = static_cast<T*>(p.out) + (int64_t)b * p.o_bstride;
  const T* nv = p.noise_vec ? static_cast<const T*>(p.noise_vec) + (int64_t)b * p.nv_bstride : nullptr;
  const bool pad_id = p.flags & GPK_KM_PAD_IDENTITY;
  const T coef = (T)p.desc.coef[0];
  uint32_t phases = 0u;  // bit b = parity the next wait on bars[b] expects

  for (int c = c_begin; c < c_end; ++c) {
    const int buf = (c - c_begin) & 1;
    const int64_t c0 = (int64_t)c * KM_TILE;
    const int yr = y_rows(c);
    T* ys = ysb + (size_t)buf * KM_TILE * d;
    if (bulk) {
      if (threadIdx.x == 0 && c + 1 < c_end) {  // prefetch the next y tile into the other buffer (freed one iteration ago)
        const uint32_t yb = (uint32_t)y_rows(c + 1) * d * sizeof(T);
        fence_proxy_async();  // the generic-proxy reads of that buffer (last tile's transposition) precede the async write
        mbar_arrive_expect_tx(&bars[buf ^ 1], yb);
        if (yb) bulk_copy_g2s(ysb + (size_t)(buf ^ 1) * KM_TILE * d, yg0 + (c0 + KM_TILE) * d, yb, &bars[buf ^ 1]);
      }
      mbar_wait(&bars[buf], (phases >> buf) & 1u);
      phases ^= 1u << buf;
    } else {
      const T* yg = yg0 + c0 * d;
      for (int i = threadIdx.x; i < yr * d; i += KM_THREADS) ys[i] = yg[i];
      __syncthreads();
    }
    // transpose the y rows to [k][64 (+1 pad)]: the 16 column-threads of a half-warp then read consecutive words
    for (int idx = threadIdx.x; idx < yr * d; idx += KM_THREADS) {
      const int cc = idx / d, k = idx - cc * d;
      yt[(size_t)k * (KM_TILE + 1) + cc] = ys[idx];
    }
    __syncthreads();

    T d2[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) d2[i][j] = T(0);
    const T* xr_ = xs + (size_t)(ty * 4) * d;
    const T* yc_ = yt + tx;
#pragma unroll 2
    for (int k = 0; k < d; ++k) {
      T xv[4], yv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) xv[i] = xr_[i * d + k];
#pragma unroll
      for (int j = 0; j < 4; ++j) yv[j] = yc_[(size_t)k * (KM_TILE + 1) + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const T df = xv[i] - yv[j];
          d2[i][j] = fma(df, df, d2[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t r = r0 + ty * 4 + i;
      if (r >= p.rows_out) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int64_t cc = c0 + tx + 16 * j;
        if (cc >= p.cols_out) continue;
        T val;
        if (r >= p.n || cc >= p.n2) {
          val = (pad_id && r == cc) ? T(1) : T(0);
        } else {
          val = coef * fast_factor<T, KIND>(d2[i][j], d, tab);
          if (same_obj && r == cc) {
            val += (T)p.noise_scalar;
            if (nv) val += nv[r];
            val += (T)p.jitter;
          }
        }
        out[r * p.ldo + cc] = val;
      }
    }
    __syncthreads();  // yt (and, without the bulk engine, ys) are rewritten by the next tile
  }
}

template <typename T, int KIND>
static int launch_fast(const KmParams& p, dim3 grid, int smem, void* stream) {
  if (const int rc = opt_in_smem<kernel_matrix_fast_kernel<T, KIND>>(smem)) return rc;
  kernel_matrix_fast_kernel<T, KIND><<<grid, KM_THREADS, smem, (cudaStream_t)stream>>>(p);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

template <typename T>
static int launch_kernel_matrix(const gpk_kernel_desc* desc, const T* xg, int64_t xg_gstride, int64_t x_bstride,
                                int64_t n, const T* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n2, int32_t d,
                                double noise_scalar, const T* noise_vec, int64_t nv_bstride, double jitter,
                                int32_t flags, T* out, int64_t ldo, int64_t o_bstride, int32_t batch, void* stream) {
  if (!desc || !xg || !yg || !out || n < 0 || n2 < 0 || d < 1 || batch < 1) return GPK_ERR_ARG;
  if (desc->n_terms < 0 || desc->n_terms > GPK_MAX_TERMS || desc->n_groups < 1 || desc->n_groups > GPK_MAX_GROUPS)
    return GPK_ERR_ARG;
  if (desc->term_begin[desc->n_terms] > GPK_MAX_FACTORS) return GPK_ERR_ARG;
  const bool pad = flags & (GPK_KM_PAD_IDENTITY | GPK_KM_PAD_ZERO);
  KmParams p;
  p.desc = *desc;
  p.xg = xg;
  p.yg = yg;
  p.xg_gstride = xg_gstride;
  p.x_bstride = x_bstride;
  p.yg_gstride = yg_gstride;
  p.y_bstride = y_bstride;
  p.n = n;
  p.n2 = n2;
  p.d = d;
  p.noise_scalar = noise_scalar;
  p.noise_vec = noise_vec;
  p.nv_bstride = nv_bstride;
  p.jitter = jitter;
  p.flags = flags;
  p.out = out;
  p.ldo = ldo;
  p.o_bstride = o_bstride;
  p.rows_out = pad ? gpk_round_up(n) : n;
  p.cols_out = pad ? gpk_round_up(n2) : n2;
  if (p.rows_out == 0 || p.cols_out == 0) return 0;
  if (ldo < p.cols_out) return GPK_ERR_ARG;
  dim3 grid((unsigned)((p.cols_out + KM_TILE - 1) / KM_TILE), (unsigned)((p.rows_out + KM_TILE - 1) / KM_TILE),
            (unsigned)batch);
  if (grid.y > 65535 || grid.z > 65535) return GPK_ERR_UNSUPPORTED;
  // one stationary factor: the specialised kernel
  const int kind0 = desc->fac_kind[0];
  if (desc->n_terms == 1 && desc->term_begin[1] - desc->term_begin[0] == 1 && kind0 >= GPK_EQ && kind0 <= GPK_MATERN52 &&
      desc->fac_group[0] >= 0 && desc->fac_group[0] < desc->n_groups) {
    // x rows, two y buffers and the transposed y tile
    const size_t fsmem = ((size_t)3 * KM_TILE * d + (size_t)d * (KM_TILE + 1)) * sizeof(T);
    if (fsmem <= 96 * 1024) {
      const dim3 fgrid((grid.x + KM_STRIP - 1) / KM_STRIP, grid.y, grid.z);
      switch (kind0) {
        case GPK_EQ: return launch_fast<T, GPK_EQ>(p, fgrid, (int)fsmem, stream);
        case GPK_MATERN12: return launch_fast<T, GPK_MATERN12>(p, fgrid, (int)fsmem, stream);
        case GPK_MATERN32: return launch_fast<T, GPK_MATERN32>(p, fgrid, (int)fsmem, stream);
        default: return launch_fast<T, GPK_MATERN52>(p, fgrid, (int)fsmem, stream);
      }
    }
  }
  const size_t smem = ((size_t)2 * desc->n_groups * KM_TILE * d + (size_t)desc->n_groups * d * (KM_TILE + 1)) * sizeof(T);
  if (smem > 200 * 1024) return GPK_ERR_UNSUPPORTED;
  if (const int rc = opt_in_smem<kernel_matrix_kernel<T>>((int)smem)) return rc;
  kernel_matrix_kernel<T><<<grid, KM_THREADS, smem, (cudaStream_t)stream>>>(p);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

int kernel_rows(const gpk_kernel_desc* desc, const double* xg, int64_t xg_gstride, int64_t n, const double* yg,
                int64_t yg_gstride, int64_t n2, int32_t d, double* out, int64_t ldo, cudaStream_t stream) {
  return launch_kernel_matrix<double>(desc, xg, xg_gstride, 0, n, yg, yg_gstride, 0, n2, d, 0.0, nullptr, 0, 0.0,
                                      GPK_KM_PAD_ZERO, out, ldo, 0, 1, stream);
}
int kernel_rows(const gpk_kernel_desc* desc, const float* xg, int64_t xg_gstride, int64_t n, const float* yg,
                int64_t yg_gstride, int64_t n2, int32_t d, float* out, int64_t ldo, cudaStream_t stream) {
  return launch_kernel_matrix<float>(desc, xg, xg_gstride, 0, n, yg, yg_gstride, 0, n2, d, 0.0, nullptr, 0, 0.0,
                                     GPK_KM_PAD_ZERO, out, ldo, 0, 1, stream);
}

// ---- elwise ------------------------------------------------------------------------------------------
struct KdParams {
  gpk_kernel_desc desc;
  const void* xg;
  const void* yg;
  int64_t xg_gstride, x_bstride, yg_gstride, y_bstride, n;
  int32_t d, same;
  void* out;
  int64_t o_bstride;
};

template <typename T>
__global__ void kernel_diag_kernel(const KdParams p) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= p.n) return;
  const T* xg = static_cast<const T*>(p.xg) + (int64_t)b * p.x_bstride;
  const T* yg = static_cast<const T*>(p.yg) + (int64_t)b * p.y_bstride;
  T acc = T(0);
  for (int t = 0; t < p.desc.n_terms; ++t) {
    T prod = (T)p.desc.coef[t];
    for (int f = p.desc.term_begin[t]; f < p.desc.term_begin[t + 1]; ++f) {
      const int g = p.desc.fac_group[f];
      const T* xr = xg + g * p.xg_gstride + i * p.d;
      const T* yr = yg + g * p.yg_gstride + i * p.d;
      T d2 = T(0), dt = T(0);
      for (int k = 0; k < p.d; ++k) {
        T df = xr[k] - yr[k];
        d2 = fma(df, df, d2);
        dt = fma(xr[k], yr[k], dt);
      }
      prod *= eval_factor<T>(p.desc.fac_kind[f], d2, dt, true, p.same != 0, p.d, p.desc.fac_param[f]);
    }
    acc += prod;
  }
  static_cast<T*>(p.out)[(int64_t)b * p.o_bstride + i] = acc;
}

template <typename T>
static int launch_kernel_diag(const gpk_kernel_desc* desc, const T* xg, int64_t xg_gstride, int64_t x_bstride,
                              const T* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n, int32_t d, int32_t same,
                              T* out, int64_t o_bstride, int32_t batch, void* stream) {
  if (!desc || !xg || !yg || !out || n < 0 || d < 1 || batch < 1) return GPK_ERR_ARG;
  if (n == 0) return 0;
  KdParams p;
  p.desc = *desc;
  p.xg = xg;
  p.yg = yg;
  p.xg_gstride = xg_gstride;
  p.x_bstride = x_bstride;
  p.yg_gstride = yg_gstride;
  p.y_bstride = y_bstride;
  p.n = n;
  p.d = d;
  p.same = same;
  p.out = out;
  p.o_bstride = o_bstride;
  dim3 grid((unsigned)((n + 255) / 256), (unsigned)batch);
  kernel_diag_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

}  // namespace gpk

extern "C" {

int gpk_kernel_matrix_f64(const gpk_kernel_desc* desc_host, const double* xg, int64_t xg_gstride, int64_t x_bstride,
                          int64_t n, const double* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n2, int32_t d,
                          double noise_scalar, const double* noise_vec, int64_t nv_bstride, double jitter,
                          int32_t flags, double* out, int64_t ldo, int64_t o_bstride, int32_t batch, void* stream) {
  return gpk::launch_kernel_matrix<double>(desc_host, xg, xg_gstride, x_bstride, n, yg, yg_gstride, y_bstride, n2, d,
                                           noise_scalar, noise_vec, nv_bstride, jitter, flags, out, ldo, o_bstride,
                                           batch, stream);
}
int gpk_kernel_matrix_f32(const gpk_kernel_desc* desc_host, const float* xg, int64_t xg_gstride, int64_t x_bstride,
                          int64_t n, const float* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n2, int32_t d,
                          double noise_scalar, const float* noise_vec, int64_t nv_bstride, double jitter,
                          int32_t flags, float* out, int64_t ldo, int64_t o_bstride, int32_t batch, void* stream) {
  return gpk::launch_kernel_matrix<float>(desc_host, xg, xg_gstride, x_bstride, n, yg, yg_gstride, y_bstride, n2, d,
                                          noise_scalar, noise_vec, nv_bstride, jitter, flags, out, ldo, o_bstride,
                                          batch, stream);
}
int gpk_kernel_diag_f64(const gpk_kernel_desc* desc_host, const double* xg, int64_t xg_gstride, int64_t x_bstride,
                        const double* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n, int32_t d, int32_t same,
                        double* out, int64_t o_bstride, int32_t batch, void* stream) {
  return gpk::launch_kernel_diag<double>(desc_host, xg, xg_gstride, x_bstride, yg, yg_gstride, y_bstride, n, d, same,
                                         out, o_bstride, batch, stream);
}
int gpk_kernel_diag_f32(const gpk_kernel_desc* desc_host, const float* xg, int64_t xg_gstride, int64_t x_bstride,
                        const float* yg, int64_t yg_gstride, int64_t y_bstride, int64_t n, int32_t d, int32_t same,
                        float* out, int64_t o_bstride, int32_t batch, void* stream) {
  return gpk::launch_kernel_diag<float>(desc_host, xg, xg_gstride, x_bstride, yg, yg_gstride, y_bstride, n, d, same,
                                        out, o_bstride, batch, stream);
}
}
