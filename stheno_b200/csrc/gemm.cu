// GEMM  C = beta*C + alpha * A * B^T  (NT: both operands K-contiguous) -- the BLAS-3 engine of the Cholesky
// trailing update (SYRK, lower tiles only), the panel updates, the recursive TRSM and the posterior covariance.
//
// fp64: warp tiles of 32 x 32 in DMMA.8x8x4 fragments (fp64 tensor cores; wgmma has no f64 type), two kernels:
//   v3  K >= 512 and K % 32 == 0 (the trailing updates): one 128 x 64 tile per CTA, 8 warps, two CTAs per SM,
//       BK = 32 x 2 stages;
//   v2  every other K: 128 x 128 tiles, 16 warps, one CTA per SM, persistent over the tiles when K < 512;
//       BK = 32 x 3 stages when K % 32 == 0, else 16 x 4.
//   Operands are staged by a cp.async (LDGSTS) ring into a FRAGMENT-MAJOR shared-memory layout: the 16-byte granule
//   holding (row, k = 2j, 2j+1) is stored where lane (row % 8) * 4 + j of the owning 8-row block reads it, so every
//   fragment load is one conflict-free, warp-contiguous LDS.128 that feeds TWO DMMAs (the even-k one and the odd-k one --
//   the k order inside a k-group of 8 is permuted identically for A and B, which leaves the product unchanged).
//   Roofline: fp64 tensor pipe (measured 37.1 TFLOP/s DMMA peak); algorithmic flops 2 M N K (M N K for lower).
//   Large batch-1 products go to the int8-slice emulation (gemm_oz.cu) instead when the caller passes its slices and scratch.
// fp32: the 3xTF32 wgmma kernel (gemm_tc32.cu) where its shape rules allow, else a register-tiled FFMA kernel (8 x 8
//   micro-tiles), double-buffered.
#include <vector>

#include "common.cuh"

namespace gpk {

constexpr int GM_BM = 128, GM_BN = 128, GM_BK = 16, GM_THREADS = 256;

template <typename T>
struct GemmParams {
  int64_t M, N, K;
  T alpha, beta;
  const T* A;
  int64_t lda, a_bs;
  const T* B;
  int64_t ldb, b_bs;
  T* C;
  int64_t ldc, c_bs;
  int32_t lower;
  int32_t tiles_m, tiles_n;
};

// CTA -> tile mapping: groups of 8 tile-rows are walked column-by-column so that concurrently resident CTAs
// share A and B panels in L2.
__device__ __forceinline__ void tile_coords(int id, int tiles_m, int tiles_n, int& tm, int& tn) {
  const int GROUP = 8;
  const int per_group = GROUP * tiles_n;
  const int group = id / per_group;
  const int first_m = group * GROUP;
  const int gsize = min(tiles_m - first_m, GROUP);
  const int r = id - group * per_group;
  tm = first_m + r % gsize;
  tn = r / gsize;
}

// ---- fp64 v2: persistent CTAs, 16 warps, operand prefetch running across tile boundaries ----------------------------
// One CTA per SM loops over the valid output tiles (static striding over a grouped rasterisation that keeps the A/B
// panels of concurrently processed tiles in L2).  The cp.async pipeline treats the CTA's whole sequence of
// (tile, k-tile) steps as ONE stream, so the operands of the next tile are already in flight while the current tile's
// last k-tiles and its epilogue run: the per-tile prologue bubble disappears (it is ~15 % of a K = 128 panel update).
// 16 warps (4 x 4, warp tile 32 x 32) put four warps on every SM sub-partition: enough independent DMMA chains to keep
// the fp64 tensor pipe busy across the per-k-tile barrier and the LDS latency (the 8-warp version idles it ~17 %).
constexpr int G2_THREADS = 512;

struct Gemm2Params {
  int64_t K;
  double alpha, beta;
  const double* A;
  int64_t lda, a_bs;
  const double* B;
  int64_t ldb, b_bs;
  double* C;
  int64_t ldc, c_bs;
  int32_t lower, tiles_m, tiles_n, n_groups;
  int32_t tiles_per_batch, total_tiles;
};

// lower mode: the valid tiles of tile rows 0 .. rows - 1 (row i holds min(i + 1, tiles_n) of them)
__host__ __device__ __forceinline__ int g2_lower_tiles(int rows, int tiles_n) {
  const int tri = rows < tiles_n ? rows : tiles_n;
  return tri * (tri + 1) / 2 + (rows - tri) * tiles_n;
}

__device__ __forceinline__ void g2_decode(const Gemm2Params& p, int idx, int& b, int& tm, int& tn) {
  b = idx / p.tiles_per_batch;
  int r = idx - b * p.tiles_per_batch;
  if (!p.lower) {
    tile_coords(r, p.tiles_m, p.tiles_n, tm, tn);
    return;
  }
  int g = 0;  // the 8-row group of tile r
  while (g + 1 < p.n_groups && g2_lower_tiles(8 * (g + 1), p.tiles_n) <= r) ++g;
  r -= g2_lower_tiles(8 * g, p.tiles_n);
  const int first = g * 8;
  const int gsize = min(p.tiles_m - first, 8);
  const int c0 = min(first, p.tiles_n);  // columns left of the group's diagonal block: all gsize rows valid
  if (r < c0 * gsize) {
    tn = r / gsize;
    tm = first + r - tn * gsize;
    return;
  }
  r -= c0 * gsize;
  for (int c = 0; c < gsize; ++c) {  // triangular part: column first + c holds rows first + c .. first + gsize - 1
    const int cnt = gsize - c;
    if (r < cnt) {
      tn = first + c;
      tm = tn + r;
      return;
    }
    r -= cnt;
  }
  tn = 0;
  tm = first;  // unreachable
}

// BK x STAGES: 16 x 4 (128 KB) or 32 x 3 (192 KB).  The deeper k-tile halves the number of barrier / wait_group /
// address-recompute episodes per flop -- ncu shows the DMMA pipe idling ~18 % of the time around them with BK = 16.
template <int BK, int STAGES>
__global__ void __launch_bounds__(G2_THREADS, 1) gemm_nt_f64_v2_kernel(const __grid_constant__ Gemm2Params p) {
  constexpr int K8 = BK / 8;                 // k8-groups per k-tile
  constexpr int STAGE_ELEMS = GM_BM * BK;    // per operand per stage
  constexpr int RB = K8 * 64;                // doubles per 8-row block
  constexpr int GPR = BK / 2;                // 16-byte granules per row
  constexpr int ROWS_PER_PASS = G2_THREADS / GPR;
  constexpr int PASSES = GM_BM / ROWS_PER_PASS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 2, wn = warp & 3;  // 4 x 4 warps; warp tile 32 x 32
  extern __shared__ __align__(16) double gm_smem[];
  double* As = gm_smem;
  double* Bs = gm_smem + STAGES * STAGE_ELEMS;

  const int KT = (int)(p.K / BK);
  const int my_tiles = (p.total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int total_iters = my_tiles * KT;

  // loader: thread copies granule ld_g of rows ld_row + ROWS_PER_PASS * i
  const int ld_row = tid / GPR, ld_g = tid % GPR;
  const int ld_off = (ld_row >> 3) * RB + ((ld_g >> 2) * 32 + (ld_row & 7) * 4 + (ld_g & 3)) * 2;
  int ld_it = 0, ld_kt = 0, ld_tile = blockIdx.x, ld_slot = 0;
  const double *ld_a = nullptr, *ld_b = nullptr;
  auto load_next = [&]() {
    if (ld_it < total_iters) {
      if (ld_kt == 0) {
        int b, tm, tn;
        g2_decode(p, ld_tile, b, tm, tn);
        ld_a = p.A + (int64_t)b * p.a_bs + ((int64_t)tm * GM_BM + ld_row) * p.lda + ld_g * 2;
        ld_b = p.B + (int64_t)b * p.b_bs + ((int64_t)tn * GM_BN + ld_row) * p.ldb + ld_g * 2;
      }
      double* as = As + ld_slot * STAGE_ELEMS + ld_off;
      double* bs = Bs + ld_slot * STAGE_ELEMS + ld_off;
      const int64_t koff = (int64_t)ld_kt * BK;
#pragma unroll
      for (int i = 0; i < PASSES; ++i) {
        cp_async16(as + i * (ROWS_PER_PASS / 8) * RB, ld_a + (int64_t)i * ROWS_PER_PASS * p.lda + koff);
        cp_async16(bs + i * (ROWS_PER_PASS / 8) * RB, ld_b + (int64_t)i * ROWS_PER_PASS * p.ldb + koff);
      }
      ++ld_it;
      if (++ld_slot == STAGES) ld_slot = 0;
      if (++ld_kt == KT) {
        ld_kt = 0;
        ld_tile += gridDim.x;
      }
    }
    cp_async_commit();
  };

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) load_next();

  double acc[4][4][2];
  int slot = 0;
  const int frag_a = (wm * 4) * RB + lane * 2, frag_b = (wn * 4) * RB + lane * 2;
  for (int t = 0; t < my_tiles; ++t) {
    int b, tm, tn;
    g2_decode(p, (int)blockIdx.x + t * (int)gridDim.x, b, tm, tn);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    for (int kt = 0; kt < KT; ++kt) {
      cp_async_wait<STAGES - 2>();
      __syncthreads();
      const double* as = As + slot * STAGE_ELEMS + frag_a;
      const double* bs = Bs + slot * STAGE_ELEMS + frag_b;
#pragma unroll
      for (int k8 = 0; k8 < K8; ++k8) {
        double2 a[4], bb[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const double2*>(as + i * RB + k8 * 64);
#pragma unroll
        for (int j = 0; j < 4; ++j) bb[j] = *reinterpret_cast<const double2*>(bs + j * RB + k8 * 64);
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) dmma884(acc[i][j][0], acc[i][j][1], a[i].x, bb[j].x);
        // refill the slot freed by the previous k-tile once the tensor pipe has work queued (not right after the
        // barrier, where it would delay the first DMMAs of all 16 warps)
        if (k8 == 0) load_next();
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) dmma884(acc[i][j][0], acc[i][j][1], a[i].y, bb[j].y);
      }
      if (++slot == STAGES) slot = 0;
    }

    double* Cg = p.C + (int64_t)b * p.c_bs + ((int64_t)tm * GM_BM + wm * 32 + (lane >> 2)) * p.ldc +
                 (int64_t)tn * GM_BN + wn * 32 + 2 * (lane & 3);
    const double alpha = p.alpha, beta = p.beta;
    if (beta != 0.0) {
      double2 old[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) old[i][j] = *reinterpret_cast<const double2*>(Cg + (int64_t)i * 8 * p.ldc + j * 8);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          double2 v;
          v.x = fma(alpha, acc[i][j][0], beta * old[i][j].x);
          v.y = fma(alpha, acc[i][j][1], beta * old[i][j].y);
          *reinterpret_cast<double2*>(Cg + (int64_t)i * 8 * p.ldc + j * 8) = v;
        }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          *reinterpret_cast<double2*>(Cg + (int64_t)i * 8 * p.ldc + j * 8) =
              make_double2(alpha * acc[i][j][0], alpha * acc[i][j][1]);
    }
  }
  cp_async_wait<0>();
}

// ---- fp64 v3: 128 x 64 tiles, 8 warps, TWO CTAs per SM ------------------------------------------------------------------
// For the large-K trailing updates.  One tile per CTA (CTAs retire continuously, so the high-priority look-ahead kernels
// get SMs), and two co-resident CTAs per SM (96 KB smem, 128 registers x 256 threads each): while one CTA sits in its
// barrier / prologue / C read-modify-write epilogue the other one keeps the DMMA pipe fed.
constexpr int G3_BN = 64, G3_THREADS = 256;

template <int BK, int STAGES>
__global__ void __launch_bounds__(G3_THREADS, 2) gemm_nt_f64_v3_kernel(const GemmParams<double> p) {
  constexpr int K8 = BK / 8;
  constexpr int RB = K8 * 64;                     // doubles per 8-row block
  constexpr int A_ELEMS = GM_BM * BK, B_ELEMS = G3_BN * BK;
  constexpr int GPR = BK / 2;                     // granules per row
  constexpr int ROWS_PER_PASS = G3_THREADS / GPR;
  constexpr int A_PASSES = GM_BM / ROWS_PER_PASS, B_PASSES = G3_BN / ROWS_PER_PASS;
  // tile mapping: p.tiles_n counts 64-wide column tiles here
  int tm, tn;
  tile_coords(blockIdx.x, p.tiles_m, p.tiles_n, tm, tn);
  if (p.lower && tn * G3_BN >= (tm + 1) * GM_BM) return;
  const int b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 1, wn = warp & 1;  // 4 x 2 warps; warp tile 32 x 32
  extern __shared__ __align__(16) double gm_smem[];
  double* As = gm_smem;
  double* Bs = gm_smem + STAGES * A_ELEMS;

  const int ld_row = tid / GPR, ld_g = tid % GPR;
  const int ld_off = (ld_row >> 3) * RB + ((ld_g >> 2) * 32 + (ld_row & 7) * 4 + (ld_g & 3)) * 2;
  const double* ld_a = p.A + (int64_t)b * p.a_bs + ((int64_t)tm * GM_BM + ld_row) * p.lda + ld_g * 2;
  const double* ld_b = p.B + (int64_t)b * p.b_bs + ((int64_t)tn * G3_BN + ld_row) * p.ldb + ld_g * 2;
  const int KT = (int)(p.K / BK);
  int ld_kt = 0, ld_slot = 0;
  auto load_next = [&]() {
    if (ld_kt < KT) {
      double* as = As + ld_slot * A_ELEMS + ld_off;
      double* bs = Bs + ld_slot * B_ELEMS + ld_off;
      const int64_t koff = (int64_t)ld_kt * BK;
#pragma unroll
      for (int i = 0; i < A_PASSES; ++i)
        cp_async16(as + i * (ROWS_PER_PASS / 8) * RB, ld_a + (int64_t)i * ROWS_PER_PASS * p.lda + koff);
#pragma unroll
      for (int i = 0; i < B_PASSES; ++i)
        cp_async16(bs + i * (ROWS_PER_PASS / 8) * RB, ld_b + (int64_t)i * ROWS_PER_PASS * p.ldb + koff);
      ++ld_kt;
      if (++ld_slot == STAGES) ld_slot = 0;
    }
    cp_async_commit();
  };
#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) load_next();

  double acc[4][4][2];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

  int slot = 0;
  const int frag_a = (wm * 4) * RB + lane * 2, frag_b = (wn * 4) * RB + lane * 2;
  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    const double* as = As + slot * A_ELEMS + frag_a;
    const double* bs = Bs + slot * B_ELEMS + frag_b;
#pragma unroll
    for (int k8 = 0; k8 < K8; ++k8) {
      double2 a[4], bb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const double2*>(as + i * RB + k8 * 64);
#pragma unroll
      for (int j = 0; j < 4; ++j) bb[j] = *reinterpret_cast<const double2*>(bs + j * RB + k8 * 64);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dmma884(acc[i][j][0], acc[i][j][1], a[i].x, bb[j].x);
      if (k8 == 0) load_next();
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dmma884(acc[i][j][0], acc[i][j][1], a[i].y, bb[j].y);
    }
    if (++slot == STAGES) slot = 0;
  }
  cp_async_wait<0>();

  double* Cg = p.C + (int64_t)b * p.c_bs + ((int64_t)tm * GM_BM + wm * 32 + (lane >> 2)) * p.ldc +
               (int64_t)tn * G3_BN + wn * 32 + 2 * (lane & 3);
  const double alpha = p.alpha, beta = p.beta;
  if (beta != 0.0) {
    double2 old[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) old[i][j] = *reinterpret_cast<const double2*>(Cg + (int64_t)i * 8 * p.ldc + j * 8);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        double2 v;
        v.x = fma(alpha, acc[i][j][0], beta * old[i][j].x);
        v.y = fma(alpha, acc[i][j][1], beta * old[i][j].y);
        *reinterpret_cast<double2*>(Cg + (int64_t)i * 8 * p.ldc + j * 8) = v;
      }
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        *reinterpret_cast<double2*>(Cg + (int64_t)i * 8 * p.ldc + j * 8) =
            make_double2(alpha * acc[i][j][0], alpha * acc[i][j][1]);
  }
}

// ---- fp32: register-tiled FFMA ------------------------------------------------------------------------
constexpr int SG_BK = 16;

__global__ void __launch_bounds__(GM_THREADS, 2) gemm_nt_f32_kernel(const GemmParams<float> p) {
  int tm, tn;
  tile_coords(blockIdx.x, p.tiles_m, p.tiles_n, tm, tn);
  if (p.lower && tn > tm) return;
  const int b = blockIdx.y;
  const int tid = threadIdx.x;
  __shared__ __align__(16) float As[2][SG_BK][GM_BM + 4];
  __shared__ __align__(16) float Bs[2][SG_BK][GM_BN + 4];

  const float* Ag = p.A + (int64_t)b * p.a_bs + (int64_t)tm * GM_BM * p.lda;
  const float* Bg = p.B + (int64_t)b * p.b_bs + (int64_t)tn * GM_BN * p.ldb;

  // global -> registers: each thread fetches 2 float4 of A and 2 of B per k-tile (128 rows x 16 k = 512 float4)
  const int lr = tid >> 2, lk = (tid & 3) * 4;  // rows lr, lr + 64; k offset lk
  float4 ra[2], rb[2];
  auto gload = [&](int kt) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      ra[i] = *reinterpret_cast<const float4*>(Ag + (int64_t)(lr + 64 * i) * p.lda + (int64_t)kt * SG_BK + lk);
      rb[i] = *reinterpret_cast<const float4*>(Bg + (int64_t)(lr + 64 * i) * p.ldb + (int64_t)kt * SG_BK + lk);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = lr + 64 * i;
      As[buf][lk + 0][r] = ra[i].x;
      As[buf][lk + 1][r] = ra[i].y;
      As[buf][lk + 2][r] = ra[i].z;
      As[buf][lk + 3][r] = ra[i].w;
      Bs[buf][lk + 0][r] = rb[i].x;
      Bs[buf][lk + 1][r] = rb[i].y;
      Bs[buf][lk + 2][r] = rb[i].z;
      Bs[buf][lk + 3][r] = rb[i].w;
    }
  };

  const int tx = tid & 15, ty = tid >> 4;  // thread tile: rows ty*4 + {0..3} and 64 + ty*4 + {0..3}; cols likewise with tx
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  const int KT = (int)(p.K / SG_BK);
  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < KT; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < KT) gload(kt + 1);
#pragma unroll
    for (int k = 0; k < SG_BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < KT) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }

  float* Cg = p.C + (int64_t)b * p.c_bs + (int64_t)tm * GM_BM * p.ldc + (int64_t)tn * GM_BN;
  const float alpha = p.alpha, beta = p.beta;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = (i < 4) ? ty * 4 + i : 64 + ty * 4 + (i - 4);
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      float4* cp = reinterpret_cast<float4*>(Cg + (int64_t)r * p.ldc + jh * 64 + tx * 4);
      float4 v;
      if (beta != 0.f) {
        const float4 o = *cp;
        v.x = fmaf(alpha, acc[i][jh * 4 + 0], beta * o.x);
        v.y = fmaf(alpha, acc[i][jh * 4 + 1], beta * o.y);
        v.z = fmaf(alpha, acc[i][jh * 4 + 2], beta * o.z);
        v.w = fmaf(alpha, acc[i][jh * 4 + 3], beta * o.w);
      } else {
        v.x = alpha * acc[i][jh * 4 + 0];
        v.y = alpha * acc[i][jh * 4 + 1];
        v.z = alpha * acc[i][jh * 4 + 2];
        v.w = alpha * acc[i][jh * 4 + 3];
      }
      *cp = v;
    }
  }
}

template <typename T>
static int check_gemm_args(int64_t M, int64_t N, int64_t K, const T* A, int64_t lda, const T* B, int64_t ldb, T* C,
                           int64_t ldc, int32_t batch) {
  if (M < 0 || N < 0 || K < 0 || batch < 1 || !A || !B || !C) return GPK_ERR_ARG;
  if (M % GM_BM || N % GM_BN || K % GM_BK) return GPK_ERR_ARG;
  if (lda < K || ldb < K || ldc < N) return GPK_ERR_ARG;
  const int64_t al = 16 / sizeof(T);
  if (lda % al || ldb % al || ldc % al) return GPK_ERR_ALIGN;
  if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(C)) % 16)
    return GPK_ERR_ALIGN;
  return 0;
}

// ---- in-situ timing of the dominant kernel (bench.py's roofline leg) ----------------------------------------------
// When enabled, every fp64 GEMM launch is bracketed by two events on ITS OWN stream; gpk_gemm_profile_read() sums the
// elapsed times and the algorithmic flops (2 * 128 * 128 * K per computed tile) after the caller has synchronised.
// kind 0: fp64 DMMA trailing-update GEMM (v3 kernel); kind 1: int8-slice emulation GEMM (gemm_oz.cu)
struct GemmProfile {
  bool enabled = false;
  std::vector<cudaEvent_t> ev;  // pairs
  std::vector<double> flops;
  std::vector<int> kind;
};
static GemmProfile g_prof;

bool prof_enabled() { return g_prof.enabled; }
void prof_begin(cudaStream_t s, double flops, int kind) {
  cudaEvent_t a, b;
  if (cudaEventCreate(&a) != cudaSuccess || cudaEventCreate(&b) != cudaSuccess) return;
  g_prof.ev.push_back(a);
  g_prof.ev.push_back(b);
  g_prof.flops.push_back(flops);
  g_prof.kind.push_back(kind);
  cudaEventRecord(a, s);
}
void prof_end(cudaStream_t s) { cudaEventRecord(g_prof.ev.back(), s); }

int gemm_nt(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, int64_t a_bs, const double* B,
            int64_t ldb, int64_t b_bs, double beta, double* C, int64_t ldc, int64_t c_bs, int32_t lower, int32_t batch,
            int32_t slices, void* ws, int64_t ws_bytes, cudaStream_t stream) {
  int rc = check_gemm_args<double>(M, N, K, A, lda, B, ldb, C, ldc, batch);
  if (!rc) rc = oz_check_emulation(slices, ws);
  if (rc) return rc;
  if (M == 0 || N == 0) return 0;
  if (batch == 1 && slices) {  // large updates: int8-slice emulation on wgmma when the caller asked for it
    rc = gemm_nt_f64_emulated(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, lower, slices, ws, ws_bytes, stream);
    if (rc < 0) return rc;
    if (rc == 1) return 0;
  }
  const int32_t tiles_m = (int32_t)(M / GM_BM), tiles_n = (int32_t)(N / GM_BN);
  if (K >= 512 && K % 32 == 0) {
    GemmParams<double> p3{M, N, K, alpha, beta, A, lda, a_bs, B, ldb, b_bs, C, ldc, c_bs, lower, tiles_m,
                          (int32_t)(N / G3_BN)};
    constexpr int smem = (GM_BM + G3_BN) * 32 * 2 * (int)sizeof(double);  // BK = 32, 2 stages: 96 KB
    if ((rc = opt_in_smem<gemm_nt_f64_v3_kernel<32, 2>>(smem))) return rc;
    dim3 grid3((unsigned)(p3.tiles_m * p3.tiles_n), (unsigned)batch);
    if (g_prof.enabled) {
      const double tn = (double)tiles_n, tmm = (double)tiles_m;
      const double tiles = lower ? (tn * (tn + 1) / 2 + (tmm - tn) * tn) : tmm * tn;  // in 128 x 128 units
      prof_begin(stream, tiles * 2.0 * GM_BM * GM_BN * (double)K * batch, 0);
    }
    gemm_nt_f64_v3_kernel<32, 2><<<grid3, G3_THREADS, smem, stream>>>(p3);
    if (g_prof.enabled) prof_end(stream);
    GPK_COUNT_LAUNCH();
    GPK_CHECK_LAUNCH();
    return 0;
  }
  if ((M / GM_BM) * (N / GM_BN) * batch >= (1ll << 30)) return GPK_ERR_UNSUPPORTED;  // v2 counts tiles in int32
  Gemm2Params q{K, alpha, beta, A, lda, a_bs, B, ldb, b_bs, C, ldc, c_bs, lower, tiles_m, tiles_n, (tiles_m + 7) / 8};
  q.tiles_per_batch = lower ? g2_lower_tiles(tiles_m, tiles_n) : tiles_m * tiles_n;
  q.total_tiles = q.tiles_per_batch * batch;
  static const int num_sms = [] {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
  }();
  constexpr int smem16 = 2 * 4 * GM_BM * 16 * (int)sizeof(double);  // BK = 16, 4 stages: 128 KB
  constexpr int smem32 = 2 * 3 * GM_BM * 32 * (int)sizeof(double);  // BK = 32, 3 stages: 192 KB
  // Small-K updates (panel steps) run persistent: the cross-tile prefetch hides their per-tile prologue.  Large-K
  // updates launch one CTA per tile instead, so that CTAs retire continuously and the high-priority look-ahead kernels
  // of the side stream can get SMs while the update is in flight.
  const int grid = (K < 512 && q.total_tiles > num_sms) ? num_sms : q.total_tiles;
  // (the in-situ profile covers the dominant kernel only -- the v3 trailing-update GEMM)
  if (K % 32 == 0) {
    if ((rc = opt_in_smem<gemm_nt_f64_v2_kernel<32, 3>>(smem32))) return rc;
    gemm_nt_f64_v2_kernel<32, 3><<<grid, G2_THREADS, smem32, stream>>>(q);
  } else {
    if ((rc = opt_in_smem<gemm_nt_f64_v2_kernel<16, 4>>(smem16))) return rc;
    gemm_nt_f64_v2_kernel<16, 4><<<grid, G2_THREADS, smem16, stream>>>(q);
  }
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

int gemm_nt(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t lda, int64_t a_bs, const float* B,
            int64_t ldb, int64_t b_bs, float beta, float* C, int64_t ldc, int64_t c_bs, int32_t lower, int32_t batch, int32_t,
            void*, int64_t, cudaStream_t stream) {
  int rc = check_gemm_args<float>(M, N, K, A, lda, B, ldb, C, ldc, batch);
  if (rc) return rc;
  if (M == 0 || N == 0) return 0;
  // tensor-core path (wgmma + TMA, 3xTF32) when the shape allows it; FFMA kernel otherwise
  rc = gemm_nt_f32_tc(M, N, K, alpha, A, lda, a_bs, B, ldb, b_bs, beta, C, ldc, c_bs, lower, batch, stream);
  if (rc < 0) return rc;
  if (rc == 1) return 0;
  GemmParams<float> p{M, N, K, alpha, beta, A, lda, a_bs, B, ldb, b_bs, C, ldc, c_bs, lower,
                      (int32_t)(M / GM_BM), (int32_t)(N / GM_BN)};
  dim3 grid((unsigned)(p.tiles_m * p.tiles_n), (unsigned)batch);
  gemm_nt_f32_kernel<<<grid, GM_THREADS, 0, stream>>>(p);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

}  // namespace gpk

extern "C" {
void gpk_gemm_profile_enable(int32_t on) {
  for (cudaEvent_t e : gpk::g_prof.ev) cudaEventDestroy(e);
  gpk::g_prof.ev.clear();
  gpk::g_prof.flops.clear();
  gpk::g_prof.kind.clear();
  gpk::g_prof.enabled = on != 0;
}
static int profile_read_kind(int kind, double* total_ms, double* total_flops, int64_t* launches) {
  double ms = 0.0, fl = 0.0;
  int64_t cnt = 0;
  const size_t n = gpk::g_prof.flops.size();
  for (size_t i = 0; i < n; ++i) {
    if (kind >= 0 && gpk::g_prof.kind[i] != kind) continue;
    float t = 0.f;
    if (const int rc = gpk::cuda_rc(cudaEventElapsedTime(&t, gpk::g_prof.ev[2 * i], gpk::g_prof.ev[2 * i + 1]))) return rc;
    ms += t;
    fl += gpk::g_prof.flops[i];
    ++cnt;
  }
  if (total_ms) *total_ms = ms;
  if (total_flops) *total_flops = fl;
  if (launches) *launches = cnt;
  return 0;
}
int gpk_gemm_profile_read(double* total_ms, double* total_flops, int64_t* launches) {
  return profile_read_kind(0, total_ms, total_flops, launches);
}
int gpk_gemm_profile_read_kind(int32_t kind, double* total_ms, double* total_flops, int64_t* launches) {
  return profile_read_kind(kind, total_ms, total_flops, launches);
}
int gpk_gemm_nt_f64(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, int64_t a_bstride,
                    const double* B, int64_t ldb, int64_t b_bstride, double beta, double* C, int64_t ldc,
                    int64_t c_bstride, int32_t lower, int32_t batch, int32_t slices, void* ws, int64_t ws_bytes,
                    void* stream) {
  return gpk::gemm_nt(M, N, K, alpha, A, lda, a_bstride, B, ldb, b_bstride, beta, C, ldc, c_bstride, lower, batch, slices,
                      ws, ws_bytes, (cudaStream_t)stream);
}
int gpk_gemm_nt_f32(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t lda, int64_t a_bstride,
                    const float* B, int64_t ldb, int64_t b_bstride, float beta, float* C, int64_t ldc,
                    int64_t c_bstride, int32_t lower, int32_t batch, void* stream) {
  return gpk::gemm_nt(M, N, K, alpha, A, lda, a_bstride, B, ldb, b_bstride, beta, C, ldc, c_bstride, lower, batch, 0,
                      nullptr, 0, (cudaStream_t)stream);
}
}
