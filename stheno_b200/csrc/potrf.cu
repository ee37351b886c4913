// K2 / K3: blocked right-looking Cholesky (lower, row-major, in place) and the recursive triangular solve.
//
//   potrf      two-level blocking: 128-wide leaf steps inside 512-wide outer panels (NB_OUTER).  Per leaf step
//                (1) potrf_leaf  : one CTA factorises the 128 x 128 diagonal block (log-det and info folded in): fp64 = the
//                                  recursive shared-memory kernel (4 x 4 sub-blocks of 32 x 32, single-warp in-register
//                                  factorisation of each diagonal sub-block, 33 us); fp32 = the register-tiled kernel
//                                  (cyclic 8 x 8 micro-tiles, one __syncthreads per column, 30 us)
//                (2) trsm_leaf   : all rows below (incl. the fused right-hand-side rows)  X L11^T = A21
//                (3) gemm (K=128): update of the rest of the outer panel
//              and per outer panel one big SYRK-style trailing update (K = 512), which carries > 90 % of the n^3/3 flops
//              at n = 16384 with C read/written once per 512 columns: on the int8 tensor cores (fp64 emulated with exact
//              integer slice products, gemm_oz.cu) when the caller passes its slices, on the fp64 tensor cores (DMMA) otherwise
//              (measured: 512 beats 256, 768, 1024 for both).  Emulated path, n_pad >= 4096: the FAR part of the trailing
//              matrix is updated once per PAIR of panels with K = 1024 (potrf_driver_pairs): half the passes over the
//              trailing matrix and half the accumulator drains per flop, the panels themselves unchanged.
//              With look-ahead the next panel is factorised on two high-priority side streams while that update runs:
//              `chain` = leaf -> 4-CTA solve of the next 128 rows -> 17-CTA update of the next diagonal block -> leaf ...
//              (everything the next leaf depends on), `bulk` = all other rows of the block column, ordered by events.
//   trsm_right recursive halving down to the 128-wide leaf; all off-diagonal work is gemm_nt with K >= 128.
//
// Right-hand sides ride along as extra ROWS below the matrix (b^T), so L^-1 b falls out of the factorisation
// itself (B.iqf_diag's triangular solve, stheno/random.py:276) -- no separate TRSV launch chain.
//
// Reference arithmetic replaced: B.cholesky / B.logdet / B.solve (stheno/random.py:274-276,
// stheno/model/observations.py:300-301,334).
#include <stdlib.h>

#include "common.cuh"

namespace gpk {

constexpr int NB = 128;

// ---- leaf Cholesky: 128 x 128 block in registers ----------------------------------------------------------
// thread (ti, tk) = (tid / 16, tid % 16) owns elements (i, k) = (ti + 16 a, tk + 16 b), a, b < 8.
template <typename T>
__global__ void __launch_bounds__(256, 1)
potrf_leaf_kernel(T* __restrict__ A, int64_t lda, int64_t a_bs, T* __restrict__ logdet, int32_t* __restrict__ info,
                  int32_t pivot_base) {
  const int bidx = blockIdx.x;
  A += (int64_t)bidx * a_bs;
  const int tid = threadIdx.x, ti = tid >> 4, tk = tid & 15;
  __shared__ T colbuf[2][NB];
  __shared__ T diag[NB];
  __shared__ T red[8];

  T acc[8][8];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b) acc[a][b] = A[(int64_t)(ti + 16 * a) * lda + tk + 16 * b];

  int buf = 0;
#pragma unroll
  for (int jb = 0; jb < 8; ++jb) {
    for (int jj = 0; jj < 16; ++jj) {
      const int j = jj + 16 * jb;
      if (tk == jj) {
#pragma unroll
        for (int a = 0; a < 8; ++a) colbuf[buf][ti + 16 * a] = acc[a][jb];
      }
      __syncthreads();
      const T djj = colbuf[buf][j];
      if (tid == 0 && !(djj > T(0))) atomicCAS(info + bidx, 0, pivot_base + j + 1);
      // 1/sqrt via the hardware reciprocal-sqrt seed (+ Newton steps, <= 1 ulp) and sqrt = d * rsqrt(d): takes the
      // IEEE sqrt + divide software sequences (~350 cycles in fp64) off the per-column critical path.
      const T inv = t_rsqrt<T>(djj);
      const T dsq = djj * inv;
      T li[8], lk[8];
#pragma unroll
      for (int a = 0; a < 8; ++a) li[a] = colbuf[buf][ti + 16 * a] * inv;
#pragma unroll
      for (int b = 0; b < 8; ++b) lk[b] = colbuf[buf][tk + 16 * b] * inv;
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        if (b < jb) continue;
        const bool col_ok = (b > jb) || (tk > jj);
#pragma unroll
        for (int a = 0; a < 8; ++a) {
          if (a < b) continue;
          const bool ok = col_ok && ((a > b) || (ti >= tk));
          if (ok) acc[a][b] -= li[a] * lk[b];
        }
      }
      if (tk == jj) {  // finalise column j of L
#pragma unroll
        for (int a = 0; a < 8; ++a) {
          const int i = ti + 16 * a;
          if (i > j) acc[a][jb] = li[a];
          else if (i == j) acc[a][jb] = dsq;
        }
      }
      if (tid == 0) diag[j] = dsq;
      buf ^= 1;
    }
  }

#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      const int i = ti + 16 * a, k = tk + 16 * b;
      if (i >= k) A[(int64_t)i * lda + k] = acc[a][b];
    }

  __syncthreads();
  if (logdet != nullptr) {
    T v = (tid < NB) ? t_log<T>(diag[tid]) : T(0);
    v = warp_sum(v);
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    if (tid == 0) {
      T s = T(0);
#pragma unroll
      for (int w = 0; w < 8; ++w) s += red[w];
      atomicAdd(logdet + bidx, T(2) * s);
    }
  }
}

// ---- recursive leaf Cholesky: the 128 x 128 block as 4 x 4 sub-blocks of 32 x 32 in shared memory ---------------------
// The flat kernel above walks 128 dependent column steps of ~360 ns each (STS -> CTA barrier -> 16 LDS -> rsqrt -> 16 DMUL ->
// up to 64 DFMA per thread): 46 us per block, all of it on the factorisation's critical path (VERDICT r1, weak #5).  Here the
// dependent chain per column is the one a single WARP needs -- shuffle of the pivot, rsqrt, one multiply, a warp-level
// broadcast of the column through shared memory, one DFMA on the next column -- and everything that is not on the chain
// (the triangular solves of the rows below a 32-block and the rank-32 updates of the blocks to its right) runs on the
// other warps, the part the next 32-block does not need even concurrently with that block's factorisation:
//   for b = 0..3:   S0  warp 0: potf2 of A_bb in registers (lane = row)      | warps 1..15: rest of the rank-32 update of step b-1
//                   S1  one thread per row below: x L_bb^T = a  (forward substitution in registers, L_bb^T broadcast)
//                   S2  all warps: rank-32 update of block column b+1 only (what S0 / S1 of the next step read)
// Arithmetic is fp64 whatever the storage type (fp32 problems: the leaf is < 2 % of the flops).
constexpr int RL_THREADS = 384;  // 12 warps: 170 registers per thread keep the 32-column factorisation of S0 out of local memory
constexpr int RL_WARPS = RL_THREADS / 32;
constexpr int RL_LD = NB + 2;  // even: rows stay 16-byte aligned for the broadcast LDS.128 of the update
constexpr int RL_SMEM = (NB * RL_LD + 32 * 32 + 32) * (int)sizeof(double);

// rank-32 update of the 32 x 32 block (r, c) with block column b:  A_rc[:, j0:j1) -= X_r X_c[j0:j1)^T ; lane = row of the block
__device__ __forceinline__ void rl_update_cols(double* S, int r, int c, int b, int j0, int j1, int lane) {
  const double* xr = S + (32 * r + lane) * RL_LD + 32 * b;
  double x[32];
#pragma unroll
  for (int k = 0; k < 32; k += 2) {
    const double2 v = *reinterpret_cast<const double2*>(xr + k);
    x[k] = v.x;
    x[k + 1] = v.y;
  }
  for (int j = j0; j < j1; ++j) {
    if (r == c && j > lane) break;  // diagonal block: only the lower triangle is ever read again (warp-uniform bound below)
    const double* xc = S + (32 * c + j) * RL_LD + 32 * b;  // same address in every lane: broadcast
    double s0 = 0.0, s1 = 0.0;
#pragma unroll
    for (int k = 0; k < 32; k += 2) {
      const double2 v = *reinterpret_cast<const double2*>(xc + k);
      s0 = fma(x[k], v.x, s0);
      s1 = fma(x[k + 1], v.y, s1);
    }
    double* o = S + (32 * r + lane) * RL_LD + 32 * c + j;
    *o -= s0 + s1;
  }
}

// measurement helper (tools/time_leaf_phases.py): when set, thread 0 of every leaf launch writes clock64() at its phase
// boundaries (start, loaded, then S0 / S1 / S2 of each 32-block, end) into this buffer
__device__ long long* g_leaf_phase_clock = nullptr;

template <typename T>
__global__ void __launch_bounds__(RL_THREADS, 1)
potrf_leaf_rec_kernel(T* __restrict__ A, int64_t lda, int64_t a_bs, T* __restrict__ logdet, int32_t* __restrict__ info,
                      int32_t pivot_base) {
  extern __shared__ __align__(16) unsigned char rl_smem[];
  double* S = reinterpret_cast<double*>(rl_smem);  // [128][RL_LD]
  double* colT = S + NB * RL_LD;                   // [32][32]: colT[j][i] = L_bb[i][j] (column j of the current diagonal block)
  double* dinv = colT + 32 * 32;                   // [32]: 1 / L_bb[j][j]
  const int bidx = blockIdx.x;
  A += (int64_t)bidx * a_bs;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  long long* const dbg = (tid == 0 && bidx == 0) ? g_leaf_phase_clock : nullptr;
  int dbg_i = 0;
  if (dbg) dbg[dbg_i++] = clock64();

  // ---- load the lower triangle (granules of two columns; the granule that straddles the diagonal is loaded whole).
  // fp64: straight global -> shared copies (cp.async, all ~11 granules of a thread in flight at once: the staged
  // register loop took 4.8k cycles, a quarter of it latency the copies now overlap)
  for (int gi = tid; gi < NB * NB / 2; gi += RL_THREADS) {
    const int row = gi >> 6, k = (gi & 63) * 2;
    if (k <= row) {
      const T* src = A + (int64_t)row * lda + k;
      if (sizeof(T) == 8) {
        cp_async16(S + row * RL_LD + k, src);
      } else {
        const float2 f = *reinterpret_cast<const float2*>(src);
        *reinterpret_cast<double2*>(S + row * RL_LD + k) = make_double2((double)f.x, (double)f.y);
      }
    }
  }
  if (sizeof(T) == 8) {
    cp_async_commit();
    cp_async_wait<0>();
  }
  __syncthreads();
  if (dbg) dbg[dbg_i++] = clock64();

  double logsum = 0.0;  // warp 0 only
#pragma unroll 1
  for (int b = 0; b < 4; ++b) {
    // ---- S0: warp 0 factorises A_bb; the other warps finish the rank-32 update of step b - 1 (blocks right of column b)
    if (warp == 0) {
      // (A square-root-free variant -- columns kept unscaled, broadcast one step ahead of the pivot chain, MUFU reciprocal
      //  + two Newton steps -- was built and measured in round 2: 32.7 us per leaf against 33.1 us for this form, i.e. the
      //  column chain is not what bounds the leaf any more; it also moved the last digits of the reference's README
      //  regression G1 (condition number ~1e16) outside its 5e-6 window, so the Cholesky form below stays.)
      double a[32];
      double diag_l = 1.0;
      const double* row = S + (32 * b + lane) * RL_LD + 32 * b;
#pragma unroll
      for (int k = 0; k < 32; k += 2) {
        const double2 v = *reinterpret_cast<const double2*>(row + k);
        a[k] = v.x;
        a[k + 1] = v.y;
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const double d = __shfl_sync(0xffffffffu, a[j], j);
        if (lane == 0 && !(d > 0.0)) atomicCAS(info + bidx, 0, pivot_base + 32 * b + j + 1);
        const double inv = rsqrt(d);
        const double l = a[j] * inv;  // lane j: sqrt(d); lanes > j: L[lane][j]; lanes < j: unused
        colT[j * 32 + lane] = l;
        if (lane == j) {
          dinv[j] = inv;
          diag_l = l;
        }
        __syncwarp();
#pragma unroll
        for (int k = j + 1; k < 32; ++k) a[k] = fma(-l, colT[j * 32 + k], a[k]);
        a[j] = l;
      }
      double* out = S + (32 * b + lane) * RL_LD + 32 * b;
#pragma unroll
      for (int k = 0; k < 32; ++k)
        if (k <= lane) out[k] = a[k];
      logsum += log(diag_l);
    } else if (b > 0) {
      // blocks (r, c), b + 1 <= c <= r <= 3, updated with block column b - 1.  ONE unit per warp, as many columns as that
      // takes: every unit re-reads its 32 x 32 row operand from shared memory (64 wavefronts), and with 2-4 column units
      // that re-read made these updates shared-memory-bandwidth bound (phase clocks, round 2: 7.1k cycles for 3 blocks
      // whose 98k FMAs need 1.5k) -- so the column ranges are as wide as the warp count allows.
      const int pb = b - 1;
      const int nblk = (4 - b) * (3 - b) / 2;  // b = 1: (2,2) (3,2) (3,3) ; b = 2: (3,3) ; b = 3: none
      if (nblk > 0) {
        const int U = (RL_WARPS - 1) / nblk;  // units per block
        const int u = warp - 1;
        if (u < U * nblk) {
          const int blk = u / U, q = u - blk * U;
          int r, c;
          if (b == 1) {
            c = (blk == 2) ? 3 : 2;
            r = (blk == 0) ? 2 : 3;
          } else {
            r = c = 3;
          }
          rl_update_cols(S, r, c, pb, (q * 32) / U, ((q + 1) * 32) / U, lane);
        }
      }
    }
    __syncthreads();
    if (dbg) dbg[dbg_i++] = clock64();
    if (b == 3) break;
    // ---- S1: rows below the diagonal block: x L_bb^T = a, one thread per row
    const int nrows = NB - 32 * (b + 1);
    if (tid < nrows) {
      double* rowp = S + (32 * (b + 1) + tid) * RL_LD + 32 * b;
      double x[32];
#pragma unroll
      for (int k = 0; k < 32; k += 2) {
        const double2 v = *reinterpret_cast<const double2*>(rowp + k);
        x[k] = v.x;
        x[k + 1] = v.y;
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        x[j] *= dinv[j];
#pragma unroll
        for (int k = j + 1; k < 32; ++k) x[k] = fma(-x[j], colT[j * 32 + k], x[k]);
      }
#pragma unroll
      for (int k = 0; k < 32; k += 2) *reinterpret_cast<double2*>(rowp + k) = make_double2(x[k], x[k + 1]);
    }
    __syncthreads();
    if (dbg) dbg[dbg_i++] = clock64();
    // ---- S2: rank-32 update of block column b + 1 (blocks (r, b + 1), r = b + 1..3): one unit per warp (see S0)
    {
      const int c = b + 1, nblk = 4 - c, U = RL_WARPS / nblk;
      if (warp < U * nblk) {
        const int blk = warp / U, q = warp - blk * U;
        rl_update_cols(S, c + blk, c, b, (q * 32) / U, ((q + 1) * 32) / U, lane);
      }
    }
    __syncthreads();
    if (dbg) dbg[dbg_i++] = clock64();
  }

  // ---- store the lower triangle
  for (int gi = tid; gi < NB * NB / 2; gi += RL_THREADS) {
    const int row = gi >> 6, k = (gi & 63) * 2;
    if (k <= row) {
      const double2 v = *reinterpret_cast<const double2*>(S + row * RL_LD + k);
      T* dst = A + (int64_t)row * lda + k;
      if (k + 1 <= row) {
        if (sizeof(T) == 8) *reinterpret_cast<double2*>(dst) = v;
        else *reinterpret_cast<float2*>(dst) = make_float2((float)v.x, (float)v.y);
      } else {
        dst[0] = (T)v.x;  // diagonal element at an even column: the element right of it belongs to the upper triangle
      }
    }
  }
  if (logdet != nullptr && warp == 0) {
    const double s = warp_sum(logsum);
    if (lane == 0) atomicAdd(logdet + bidx, (T)(2.0 * s));
  }
  if (dbg) dbg[dbg_i++] = clock64();
}

// ---- leaf TRSM of gpk_trsm_right_t:  X L = B  (B: rows x 128, 64 rows per CTA), in place, by backward substitution
// (L lower-triangular).  Thread (r, cg) = (tid % 64, tid / 64) owns row r, columns 32 cg .. 32 cg + 31 in registers.
constexpr int TL_LD = NB + 2;

template <typename T>
__global__ void __launch_bounds__(256, 1)
trsm_leaf_kernel(const T* __restrict__ L, int64_t ldl, int64_t l_bs, T* __restrict__ B, int64_t ldb, int64_t b_bs) {
  extern __shared__ __align__(16) unsigned char tl_smem[];
  T* Lt = reinterpret_cast<T*>(tl_smem);  // Lt[j][k] = L[j][k]   (ld = TL_LD)
  T* invd = Lt + NB * TL_LD;              // 1 / L[j][j]
  T* xbuf = invd + NB;                    // [2][64]
  const int tid = threadIdx.x;
  const int bidx = blockIdx.y;
  L += (int64_t)bidx * l_bs;
  B += (int64_t)bidx * b_bs + (int64_t)blockIdx.x * 64 * ldb;

  for (int idx = tid; idx < NB * NB; idx += 256) {
    const int k = idx >> 7, j = idx & 127;  // read L[k][j] coalesced in j
    const T v = (j <= k) ? L[(int64_t)k * ldl + j] : T(0);
    Lt[k * TL_LD + j] = v;
    if (j == k) invd[j] = T(1) / v;
  }
  const int r = tid & 63, cg = tid >> 6;
  T a[32];
  {
    const T* src = B + (int64_t)r * ldb + 32 * cg;
#pragma unroll
    for (int q = 0; q < 32; ++q) a[q] = src[q];
  }
  __syncthreads();

  int buf = 0;
  for (int step = 0; step < NB; ++step) {
    const int j = NB - 1 - step;
    const int cgj = j >> 5, jj = j & 31;
    if (cg == cgj) {
      T x = T(0);
#pragma unroll
      for (int q = 0; q < 32; ++q) x = (q == jj) ? a[q] : x;
      x *= invd[j];
#pragma unroll
      for (int q = 0; q < 32; ++q) a[q] = (q == jj) ? x : a[q];
      xbuf[buf * 64 + r] = x;
    }
    __syncthreads();
    if (cg <= cgj) {
      const T x = xbuf[buf * 64 + r];
      // a[k] -= x * L[j][k] (k < j) = Lt[j][k]
      const T* lrow = Lt + j * TL_LD + 32 * cg;
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        const bool ok = (cg != cgj) || (q < jj);
        if (ok) a[q] -= x * lrow[q];
      }
    }
    buf ^= 1;
  }
  {
    T* dst = B + (int64_t)r * ldb + 32 * cg;
#pragma unroll
    for (int q = 0; q < 32; ++q) dst[q] = a[q];
  }
}

// ---- fp64 leaf TRSM on the tensor cores:  X L^T = B  (128 rows per CTA, 16 warps, 8 rows per warp) -------------
// Rows of a right-side TRSM are independent, so every warp solves its own 8 rows with NO inter-warp
// synchronisation: the 8 x 128 row block lives in registers as sixteen 8 x 8 DMMA accumulator fragments.  L11 sits in
// shared memory in the B-operand fragment-major layout of gemm.cu, with each 16 x 16 diagonal block replaced by its
// inverse.  For each 16-column block jb:   X_jb = A_jb * inv(L_jb,jb)^T ;   A[:, later] -= X_jb * L[later, jb]^T .
// The accumulator fragment of an 8 x 8 block (lane holds columns 2q, 2q+1 of row lane/4) IS the A-operand fragment
// pair of the k-permuted DMMA convention used throughout (even-k DMMA takes .x, odd-k DMMA takes .y), so results feed
// the next product straight from registers.  256 DMMA + 128 LDS.128 per warp; no shared-memory traffic for A at all.
constexpr int TC_ROWS = 128;
constexpr int TC_THREADS = 512;
constexpr int TC_SMEM = (NB * NB + 8 * 16 * 17) * (int)sizeof(double);  // L11 fragment-major + the diagonal blocks

__device__ __forceinline__ int frag_index(int n, int k) {
  // element (row n, col k) of a 128 x 128 operand in fragment-major layout (16 k8-groups per 8-row block)
  return (((n >> 3) * 16 + (k >> 3)) * 32 + (n & 7) * 4 + ((k & 7) >> 1)) * 2 + (k & 1);
}

// T = storage type (double or float).  The arithmetic is always fp64 on the DMMA pipe: for fp32 problems the leaf TRSM is
// < 2 % of the flops, and doing it in fp64 costs nothing while removing one source of fp32 round-off.
template <typename T>
__global__ void __launch_bounds__(TC_THREADS, 1)
trsm_leaf_tc_kernel(const T* __restrict__ L, int64_t ldl, int64_t l_bs, T* __restrict__ B, int64_t ldb, int64_t b_bs,
                    int32_t rows_per_cta) {
  extern __shared__ __align__(16) unsigned char tc_smem[];
  double* Ls = reinterpret_cast<double*>(tc_smem);  // 128 x 128 fragment-major
  double* Ld = Ls + NB * NB;                         // [8][16][17] diagonal blocks (natural layout)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  L += (int64_t)blockIdx.y * l_bs;
  B += (int64_t)blockIdx.y * b_bs + (int64_t)blockIdx.x * rows_per_cta * ldb;

  // (1) L11 (lower part, zeros above) -> fragment-major shared memory; 8192 granules of 2 doubles
#pragma unroll
  for (int gi = tid; gi < NB * NB / 2; gi += TC_THREADS) {  // 16 independent 2-element loads in flight per thread
    const int c = gi >> 6, g = gi & 63;  // row c, granule g: columns 2g, 2g+1
    const int k = 2 * g;
    double2 v = make_double2(0.0, 0.0);
    if (k <= c) {
      const T* src = L + (int64_t)c * ldl + k;  // (k even, ldl even, L 16-byte aligned: one vector load)
      if (sizeof(T) == 8) {
        v = *reinterpret_cast<const double2*>(src);
      } else {
        const float2 f = *reinterpret_cast<const float2*>(src);
        v = make_double2((double)f.x, (double)f.y);
      }
      if (k + 1 > c) v.y = 0.0;
    }
    *reinterpret_cast<double2*>(Ls + frag_index(c, k)) = v;
    if ((c >> 4) == (k >> 4)) {  // diagonal 16 x 16 block: natural copy for the inversion
      double* d = Ld + ((c >> 4) * 16 + (c & 15)) * 17 + (k & 15);
      d[0] = v.x;
      d[1] = v.y;
    }
  }
  __syncthreads();
  // (2) invert the eight diagonal blocks: warp d, lane c (< 16) solves L_d x = e_c by forward substitution
  //     (one reciprocal per diagonal entry, shared through the padding column of Ld; no divisions on the chain)
  if (warp < 8) {
    double* Lb = Ld + warp * 16 * 17;
    if (lane < 16) Lb[lane * 17 + 16] = 1.0 / Lb[lane * 17 + lane];
    __syncwarp();
    if (lane < 16) {
      double x[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        double s = (i == lane) ? 1.0 : 0.0;
#pragma unroll
        for (int k = 0; k < 16; ++k)
          if (k < i) s -= Lb[i * 17 + k] * x[k];
        x[i] = (i >= lane) ? s * Lb[i * 17 + 16] : 0.0;
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) Ls[frag_index(warp * 16 + i, warp * 16 + lane)] = x[i];
    }
  }
  __syncthreads();

  // (3) this warp's 8 rows as sixteen accumulator fragments.  (With rows_per_cta < 128 -- the latency-critical launches of
  //     the factorisation chain spread 128 rows over 4 CTAs -- only the first rows_per_cta / 8 warps have rows: the solve
  //     is bound by the DMMA rate of ONE SM, 11 us for 128 rows.)
  if (warp * 8 >= rows_per_cta) return;
  double acc[16][2];
  T* Bw = B + (int64_t)(warp * 8 + (lane >> 2)) * ldb + 2 * (lane & 3);
#pragma unroll
  for (int cb = 0; cb < 16; ++cb) {
    acc[cb][0] = (double)Bw[cb * 8];
    acc[cb][1] = (double)Bw[cb * 8 + 1];
  }
  const double* Lf = Ls + lane * 2;  // fragment (row block rb, k8 group kg) at Lf + (rb * 16 + kg) * 64
#pragma unroll
  for (int jb = 0; jb < 8; ++jb) {
    double x[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
#pragma unroll
    for (int nb = 0; nb < 2; ++nb)
#pragma unroll
      for (int kg = 0; kg < 2; ++kg) {
        if (kg > nb) continue;  // the inverse block is lower triangular: its (nb=0, kg=1) 8 x 8 block is zero
        const double2 b = *reinterpret_cast<const double2*>(Lf + ((2 * jb + nb) * 16 + 2 * jb + kg) * 64);
        dmma884(x[nb][0], x[nb][1], acc[2 * jb + kg][0], b.x);
        dmma884(x[nb][0], x[nb][1], acc[2 * jb + kg][1], b.y);
      }
    acc[2 * jb][0] = x[0][0];
    acc[2 * jb][1] = x[0][1];
    acc[2 * jb + 1][0] = x[1][0];
    acc[2 * jb + 1][1] = x[1][1];
    const double nx[2][2] = {{-x[0][0], -x[0][1]}, {-x[1][0], -x[1][1]}};
    // four passes (k-group x parity) over all later column blocks: consecutive DMMAs hit different accumulators
#pragma unroll
    for (int kg = 0; kg < 2; ++kg) {
      double2 b[16];
#pragma unroll
      for (int cb = 2 * jb + 2; cb < 16; ++cb)
        b[cb] = *reinterpret_cast<const double2*>(Lf + (cb * 16 + 2 * jb + kg) * 64);
#pragma unroll
      for (int cb = 2 * jb + 2; cb < 16; ++cb) dmma884(acc[cb][0], acc[cb][1], nx[kg][0], b[cb].x);
#pragma unroll
      for (int cb = 2 * jb + 2; cb < 16; ++cb) dmma884(acc[cb][0], acc[cb][1], nx[kg][1], b[cb].y);
    }
  }
#pragma unroll
  for (int cb = 0; cb < 16; ++cb) {
    Bw[cb * 8] = (T)acc[cb][0];
    Bw[cb * 8 + 1] = (T)acc[cb][1];
  }
}

// X L^T = B against a 128 x 128 leaf L, 128 rows of B per CTA: rows must be a multiple of 128
template <typename T>
static int trsm_leaf_fwd(const T* L, int64_t ldl, int64_t l_bs, T* B, int64_t ldb, int64_t b_bs, int64_t rows,
                         int32_t batch, cudaStream_t stream) {
  if (rows % TC_ROWS) return GPK_ERR_ARG;
  if (rows == 0) return 0;
  if (const int rc = opt_in_smem<trsm_leaf_tc_kernel<T>>(TC_SMEM)) return rc;
  dim3 grid((unsigned)(rows / TC_ROWS), (unsigned)batch);
  trsm_leaf_tc_kernel<T><<<grid, TC_THREADS, TC_SMEM, stream>>>(L, ldl, l_bs, B, ldb, b_bs, TC_ROWS);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

// ---- rank-128 update of one 128 x 128 diagonal block, D -= X X^T (lower 8 x 8 blocks), spread over 17 CTAs: one warp per
// 8 x 8 output block, both operands read straight from X in global memory (L2) in DMMA fragment order.  Latency-critical:
// it sits between two leaf factorisations on the chain, where a single-SM tile update would cost ~12 us.
template <typename T>
__global__ void __launch_bounds__(256)
diag_syrk_kernel(const T* __restrict__ X, int64_t ldx, int64_t x_bs, T* __restrict__ D, int64_t ldd, int64_t d_bs) {
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * 8 + (threadIdx.x >> 5);  // 0 .. 135: lower-triangular block index
  int rb = (int)((sqrtf(8.f * (float)g + 1.f) - 1.f) * 0.5f);
  while (rb * (rb + 1) / 2 > g) --rb;
  while ((rb + 1) * (rb + 2) / 2 <= g) ++rb;
  const int cb = g - rb * (rb + 1) / 2;
  X += (int64_t)blockIdx.y * x_bs;
  D += (int64_t)blockIdx.y * d_bs;
  const T* Xa = X + (int64_t)(rb * 8 + (lane >> 2)) * ldx + 2 * (lane & 3);
  const T* Xb = X + (int64_t)(cb * 8 + (lane >> 2)) * ldx + 2 * (lane & 3);
  double a[16][2], b[16][2];
#pragma unroll
  for (int kg = 0; kg < 16; ++kg) {
    a[kg][0] = (double)Xa[kg * 8];
    a[kg][1] = (double)Xa[kg * 8 + 1];
    b[kg][0] = (double)Xb[kg * 8];
    b[kg][1] = (double)Xb[kg * 8 + 1];
  }
  T* Dp = D + (int64_t)(rb * 8 + (lane >> 2)) * ldd + cb * 8 + 2 * (lane & 3);
  const double c0 = (double)Dp[0], c1 = (double)Dp[1];
  double d0[2] = {0.0, 0.0}, d1[2] = {0.0, 0.0};
#pragma unroll
  for (int kg = 0; kg < 8; ++kg) {  // two independent DMMA chains
    dmma884(d0[0], d0[1], a[kg][0], b[kg][0]);
    dmma884(d1[0], d1[1], a[kg + 8][0], b[kg + 8][0]);
    dmma884(d0[0], d0[1], a[kg][1], b[kg][1]);
    dmma884(d1[0], d1[1], a[kg + 8][1], b[kg + 8][1]);
  }
  Dp[0] = (T)(c0 - (d0[0] + d1[0]));
  Dp[1] = (T)(c1 - (d0[1] + d1[1]));
}

// The dependency of the next leaf in two short launches: the 128 rows below L11 solved by 4 CTAs (32 rows each), then the
// next diagonal block updated by 17 CTAs.
template <typename T>
static int launch_diag_step(const T* L, int64_t ldl, int64_t l_bs, T* B, int64_t ldb, int64_t b_bs, T* D, int64_t ldd,
                            int64_t d_bs, int32_t batch, cudaStream_t stream) {
  if (const int rc = opt_in_smem<trsm_leaf_tc_kernel<T>>(TC_SMEM)) return rc;
  trsm_leaf_tc_kernel<T><<<dim3(4, (unsigned)batch), TC_THREADS, TC_SMEM, stream>>>(L, ldl, l_bs, B, ldb, b_bs, 32);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  diag_syrk_kernel<T><<<dim3(17, (unsigned)batch), 256, 0, stream>>>(B, ldb, b_bs, D, ldd, d_bs);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

template <typename T>
static int launch_potrf_leaf(T* A, int64_t lda, int64_t a_bs, T* logdet, int32_t* info, int32_t pivot_base,
                             int32_t batch, cudaStream_t stream) {
  // (A DMMA-blocked leaf -- 16-column blocks, one warp factorising the 16 x 16 diagonal block with shuffles -- was
  //  built and measured at 72-170 us per block against 46 us for this register-tiled kernel: a single warp cannot
  //  retire the 16 x 16 step's dependent instruction stream fast enough.
  //  A two-columns-per-barrier (rank-2) variant measured the same: the leaf is bound by its dependent
  //  STS -> barrier -> LDS -> rsqrt -> DMUL -> DFMA chain, not by the barrier count or the fp64 pipe.)
  // fp32 storage keeps the round-1 register-tiled kernel (fp32 arithmetic, measured 29.6 us against 33.6 us for the
  // recursive one, which computes in fp64)
  if constexpr (sizeof(T) == 4) {
    potrf_leaf_kernel<T><<<batch, 256, 0, stream>>>(A, lda, a_bs, logdet, info, pivot_base);
  } else {
    if (const int rc = opt_in_smem<potrf_leaf_rec_kernel<T>>(RL_SMEM)) return rc;
    potrf_leaf_rec_kernel<T><<<batch, RL_THREADS, RL_SMEM, stream>>>(A, lda, a_bs, logdet, info, pivot_base);
  }
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

template <typename T>
static int launch_trsm_leaf(const T* L, int64_t ldl, int64_t l_bs, T* B, int64_t ldb, int64_t b_bs, int64_t rows,
                            int32_t batch, cudaStream_t stream) {
  if (rows == 0) return 0;
  const int smem = (NB * TL_LD + NB + 2 * 64) * (int)sizeof(T);
  if (const int rc = opt_in_smem<trsm_leaf_kernel<T>>(smem)) return rc;
  dim3 grid((unsigned)(rows / 64), (unsigned)batch);
  trsm_leaf_kernel<T><<<grid, 256, smem, stream>>>(L, ldl, l_bs, B, ldb, b_bs);
  GPK_COUNT_LAUNCH();
  GPK_CHECK_LAUNCH();
  return 0;
}

constexpr int64_t NB_OUTER = 512;  // outer panel width

// GPK_NO_LOOKAHEAD (read at every factorisation): the look-ahead schedule on the caller's stream alone, so that
// event-bracketed launches time single kernels (bench.py's in-situ kernel timing)
static bool no_lookahead() { return getenv("GPK_NO_LOOKAHEAD") != nullptr; }

// Side streams + events for the look-ahead, one set per (host thread, device) (`lookahead()`): concurrent factorisations on
// different host threads never share them.  Every use forks them from the caller's stream with an event and joins them
// back before the call returns, so a factorisation is ordered on the caller's stream like any single launch.
struct Lookahead {
  cudaStream_t side = nullptr;  // the latency-bound chain: leaf factorisations + the rows the next leaf depends on
  cudaStream_t bulk = nullptr;  // the rest of the panel rows (throughput work the chain does not wait for)
  cudaEvent_t fork = nullptr, join = nullptr, leaf = nullptr, crit = nullptr, bulk_done = nullptr;
  bool ok = false;
  Lookahead() {
    int lo = 0, hi = 0;
    if (cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess) return;
    if (cudaStreamCreateWithPriority(&side, cudaStreamNonBlocking, hi) != cudaSuccess) return;
    if (cudaStreamCreateWithPriority(&bulk, cudaStreamNonBlocking, hi) != cudaSuccess) return;
    for (cudaEvent_t* e : {&fork, &join, &leaf, &crit, &bulk_done})
      if (cudaEventCreateWithFlags(e, cudaEventDisableTiming) != cudaSuccess) return;
    ok = true;
  }
};

static Lookahead& lookahead() {
  // one side stream per (host thread, device): the stream must live on the device the caller's stream belongs to
  static thread_local Lookahead* la[64] = {nullptr};
  int dev = 0;
  cudaGetDevice(&dev);
  dev = (dev < 0 || dev >= 64) ? 0 : dev;
  if (la[dev] == nullptr) la[dev] = new Lookahead();
  return *la[dev];
}

// Factorise the outer panel [kb, ke): leaf Cholesky, leaf TRSM of all rows below, rank-128 update of the rest of
// the panel -- for every 128-wide step.
template <typename T>
static int factor_panel(T* A, int64_t lda, int64_t a_bs, int64_t R, int64_t kb, int64_t ke, T* logdet, int32_t* info,
                        int32_t batch, cudaStream_t stream) {
  int rc;
  for (int64_t j = kb; j < ke; j += NB) {
    T* Ajj = A + j * lda + j;
    if ((rc = launch_potrf_leaf<T>(Ajj, lda, a_bs, logdet, info, (int32_t)j, batch, stream))) return rc;
    const int64_t below = R - (j + NB);
    if (below > 0) {
      T* A21 = A + (j + NB) * lda + j;
      if ((rc = trsm_leaf_fwd<T>(Ajj, lda, a_bs, A21, lda, a_bs, below, batch, stream))) return rc;
      const int64_t ncols = ke - (j + NB);
      if (ncols > 0) {
        if ((rc = gemm_nt(below, ncols, (int64_t)NB, T(-1), A21, lda, a_bs, A21, lda, a_bs, T(1),
                          A + (j + NB) * lda + (j + NB), lda, a_bs, 1, batch, 0, nullptr, 0, stream)))
          return rc;
      }
    }
  }
  return 0;
}

// The same factorisation with the dependency chain cut short.  The next leaf only depends on the next 128 x 128 diagonal
// block, so `chain` runs  leaf -> diag_step (solve the 128 rows below the leaf, then update the next diagonal block)
// -> leaf -> ...  while every other row of the block column (the rest of the panel's diagonal block and all the
// rows below it: the throughput work) is solved / updated on the `bulk` stream, ordered by events:
//   bulk(j)  waits for leaf(j) (solve) and diag_step(j) (its rows are the B operand of the update);
//   diag_step(j + 128) waits for bulk(j) (which updated the rows it solves).
// On return `chain` has also waited for `bulk`.
template <typename T>
static int factor_panel_split(T* A, int64_t lda, int64_t a_bs, int64_t R, int64_t kb, int64_t ke, T* logdet, int32_t* info,
                              int32_t batch, cudaStream_t chain, Lookahead& la) {
  int rc;
  bool bulk_pending = false;  // bulk work the next diag_step has to wait for
  for (int64_t j = kb; j < ke; j += NB) {
    T* Ajj = A + j * lda + j;
    if ((rc = launch_potrf_leaf<T>(Ajj, lda, a_bs, logdet, info, (int32_t)j, batch, chain))) return rc;
    const int64_t j1 = j + NB;           // next diagonal block
    const bool has_next = j1 < ke;       // ... inside this panel
    const int64_t b0 = has_next ? j1 + NB : j1;  // first row the bulk stream handles
    const int64_t brows = R - b0;
    if (brows > 0) {
      if ((rc = cuda_rc(cudaEventRecord(la.leaf, chain)))) return rc;
      if ((rc = cuda_rc(cudaStreamWaitEvent(la.bulk, la.leaf, 0)))) return rc;
      if ((rc = trsm_leaf_fwd<T>(Ajj, lda, a_bs, A + b0 * lda + j, lda, a_bs, brows, batch, la.bulk))) return rc;
    }
    if (has_next) {
      if (bulk_pending) {  // the rows this step solves were updated by the previous step's bulk GEMM
        if ((rc = cuda_rc(cudaStreamWaitEvent(chain, la.bulk_done, 0)))) return rc;
      }
      T* X1 = A + j1 * lda + j;  // rows [j1, j1 + 128) of this block column
      if ((rc = launch_diag_step<T>(Ajj, lda, a_bs, X1, lda, a_bs, A + j1 * lda + j1, lda, a_bs, batch, chain))) return rc;
      if (brows > 0) {
        if ((rc = cuda_rc(cudaEventRecord(la.crit, chain)))) return rc;
        if ((rc = cuda_rc(cudaStreamWaitEvent(la.bulk, la.crit, 0)))) return rc;
        // rows [b0, R) x columns [j1, ke) of the panel -= X[b0:, j] X[j1:ke, j]^T
        if ((rc = gemm_nt(brows, ke - j1, (int64_t)NB, T(-1), A + b0 * lda + j, lda, a_bs, X1, lda, a_bs, T(1),
                          A + b0 * lda + j1, lda, a_bs, 0, batch, 0, nullptr, 0, la.bulk)))
          return rc;
        if ((rc = cuda_rc(cudaEventRecord(la.bulk_done, la.bulk)))) return rc;
        bulk_pending = true;
      }
    }
  }
  if (R - ke > 0 || bulk_pending) {
    if ((rc = cuda_rc(cudaEventRecord(la.bulk_done, la.bulk)))) return rc;
    if ((rc = cuda_rc(cudaStreamWaitEvent(chain, la.bulk_done, 0)))) return rc;
  }
  return 0;
}

// Right-looking over 1024-wide outer panels WITH LOOK-AHEAD: the trailing update of panel i is split into
// (a) the columns of panel i+1 and (b) everything to the right of it; as soon as (a) is done the latency-bound
// factorisation of panel i+1 runs on a high-priority side stream while the tensor-core-bound update (b) keeps the
// SMs busy on the caller's stream.

// How the K = NB_OUTER trailing updates of an fp64 factorisation are formed:
//   MODE_F64     fp64 tensor cores (DMMA) straight from the matrix
//   MODE_TF32X3  opt-in: fp32 copy of the panel, 3xTF32 products on wgmma (fp32-level products)
//   MODE_OZAKI   int8 slices of the panel (error-free split), exact int32 products on wgmma, fp64 recombination
enum { MODE_F64 = 0, MODE_TF32X3 = 1, MODE_OZAKI = 2 };
// scratch of the pair scheme: the pair's rows sliced 1024 wide + one panel's rows sliced 512 wide.  (Slicing the NEXT pair's
// operand on the side stream into a second 1024-wide buffer, off the caller's stream, was measured slower: 22.4 vs 21.9 ms.)
static inline int64_t potrf_pairs_ws_bytes(int64_t R, int32_t S) {
  return ((oz_ws_bytes(R, 1024, S) + 1023) & ~int64_t(1023)) + oz_ws_bytes(R, 512, S);
}
struct Trailing {
  int mode = MODE_F64;
  void* ws = nullptr;
  int64_t ws_bytes = 0;
  int32_t slices = 0;
  int64_t cap_rows = 0;  // MODE_OZAKI: rows the workspace was laid out for
};

// Prepare the workspace copy of the panel rows [row0, row0 + rows) x [kb, kb + K) (row `i` of the copy = matrix row
// row0 + i).  Returns the mode actually used for this panel.
template <typename T>
static int prepare_panel(const Trailing&, const T*, int64_t, int64_t, int64_t, int32_t, cudaStream_t, int* used) {
  *used = MODE_F64;
  return 0;
}
template <>
int prepare_panel<double>(const Trailing& t, const double* P, int64_t ldp, int64_t rows, int64_t K, int32_t batch,
                          cudaStream_t s, int* used) {
  *used = MODE_F64;
  if (t.mode == MODE_TF32X3 && batch == 1 && K % 32 == 0 && K >= 128 && t.ws_bytes >= rows * K * 4) {
    *used = MODE_TF32X3;
    return convert_panel_f32(P, ldp, rows, K, static_cast<float*>(t.ws), s);
  }
  if (t.mode == MODE_OZAKI && batch == 1 && K % 128 == 0 && rows <= t.cap_rows &&
      t.ws_bytes >= oz_ws_bytes(t.cap_rows, K, t.slices)) {
    *used = MODE_OZAKI;
    return oz_slice_panel(P, ldp, rows, K, t.ws, t.cap_rows, t.slices, s);
  }
  return 0;
}

// trailing update C[M x N] -= P[rA : rA + M] P[rB : rB + N]^T (lower: only the tiles that touch the lower triangle);
// rA / rB = first row of the operands relative to the first row of the prepared panel copy, PA / PB the same rows in
// the matrix itself.
template <typename T>
static int trailing_update(int used, const Trailing&, int64_t rA, int64_t rB, int64_t M, int64_t N, int64_t K, const T* PA,
                           const T* PB, int64_t lda, int64_t a_bs, T* C, int32_t lower, int32_t batch, cudaStream_t stream) {
  return gemm_nt(M, N, K, T(-1), PA, lda, a_bs, PB, lda, a_bs, T(1), C, lda, a_bs, lower, batch, 0, nullptr, 0, stream);
}
template <>
int trailing_update<double>(int used, const Trailing& t, int64_t rA, int64_t rB, int64_t M, int64_t N, int64_t K,
                            const double* PA, const double* PB, int64_t lda, int64_t a_bs, double* C, int32_t lower,
                            int32_t batch, cudaStream_t stream) {
  if (used == MODE_TF32X3 && rA == rB && lower)
    return syrk_f64_tf32x3(M, N, K, static_cast<const float*>(t.ws) + rA * K, C, lda, stream);
  if (used == MODE_OZAKI)
    return oz_gemm_sliced(M, N, K, -1.0, t.ws, t.cap_rows, rA, t.ws, t.cap_rows, rB, 1.0, C, lda, lower, t.slices, stream);
  return gemm_nt(M, N, K, -1.0, PA, lda, a_bs, PB, lda, a_bs, 1.0, C, lda, a_bs, lower, batch, 0, nullptr, 0, stream);
}

// ---- fp64 + int8 emulation, single matrix: outer panels factorised in PAIRS ------------------------------------------
// The emulated update drains S accumulators per 128 x 64 tile whatever K is, and every outer step reads and writes the
// whole trailing matrix once.  Widening the outer panel to 1024 directly pushes twice the rank-128 DMMA updates of the
// 128-wide leaf steps through the panel.
// Here the 512-wide panels keep their leaf steps, but the FAR part of the trailing matrix is updated once per PAIR of
// panels with K = 1024 (the pair's rows re-sliced as one 1024-wide operand), i.e. half the passes over the trailing
// matrix and half the accumulator drains per flop:
//   pair (A, B) factorised  ->  X = slices of rows below x [A | B]  (K = 1024)
//   side streams: block column A' of the next pair  -= X X^T ; factor A' ; Y = slices of rows below x A' (K = 512) ;
//                 block column B' -= X X^T (bulk stream, any time) and -= Y Y^T (after it) ; factor B'
//   caller's stream: everything right of the next pair -= X X^T (K = 1024), concurrently.
// Updates that touch the same block are ordered by streams / events (never concurrent: results stay bit-reproducible).
static int potrf_driver_pairs(double* A, int64_t lda, int64_t n_pad, int64_t extra_rows, double* logdet, int32_t* info,
                              cudaStream_t stream, void* ws, int32_t S, Lookahead& la) {
  const int64_t R = n_pad + extra_rows, P = NB_OUTER;
  const bool nola = no_lookahead();  // the same schedule on ONE stream
  const cudaStream_t side = nola ? stream : la.side, bulk = nola ? stream : la.bulk;
  auto factor = [&](int64_t c0, int64_t c1) -> int {
    if (nola) return factor_panel<double>(A, lda, 0, R, c0, c1, logdet, info, 1, stream);
    return factor_panel_split<double>(A, lda, 0, R, c0, c1, logdet, info, 1, side, la);  // ends joined with bulk
  };
  void* wsX = ws;                                                                       // [S][R][1024] + scales
  void* wsY = static_cast<char*>(ws) + ((oz_ws_bytes(R, 2 * P, S) + 1023) & ~int64_t(1023));  // [S][R][512] + scales
  int rc;
  auto upd = [&](void* w, int64_t K, int64_t rA, int64_t rB, int64_t M, int64_t N, double* C, int32_t lower,
                 cudaStream_t s) -> int {
    if (M <= 0 || N <= 0) return 0;
    return oz_gemm_sliced(M, N, K, -1.0, w, R, rA, w, R, rB, 1.0, C, lda, lower, S, s);
  };
  // first pair: panel A0, its update of B0, panel B0 -- nothing to overlap with yet
  const int64_t a1 = P < n_pad ? P : n_pad, b1 = 2 * P < n_pad ? 2 * P : n_pad;
  if ((rc = factor_panel<double>(A, lda, 0, R, 0, a1, logdet, info, 1, stream))) return rc;
  if (b1 > a1) {
    if ((rc = oz_slice_panel(A + a1 * lda, lda, R - a1, a1, wsY, R, S, stream))) return rc;
    if ((rc = upd(wsY, a1, 0, 0, R - a1, b1 - a1, A + a1 * lda + a1, 1, stream))) return rc;
    if ((rc = factor_panel<double>(A, lda, 0, R, a1, b1, logdet, info, 1, stream))) return rc;
  }
  for (int64_t kb = 0; kb + 2 * P < n_pad; kb += 2 * P) {
    const int64_t ke = kb + 2 * P;                                   // pair [kb, ke) is factorised
    const int64_t ke1 = ke + P < n_pad ? ke + P : n_pad;              // A' = [ke, ke1)
    const int64_t ke2 = ke + 2 * P < n_pad ? ke + 2 * P : n_pad;      // B' = [ke1, ke2) (may be empty)
    const int64_t W1 = ke1 - ke, W2 = ke2 - ke1, K2 = 2 * P;
    if ((rc = oz_slice_panel(A + ke * lda + kb, lda, R - ke, K2, wsX, R, S, stream))) return rc;
    if ((rc = cuda_rc(cudaEventRecord(la.fork, stream)))) return rc;
    if ((rc = cuda_rc(cudaStreamWaitEvent(side, la.fork, 0)))) return rc;
    if ((rc = cuda_rc(cudaStreamWaitEvent(bulk, la.fork, 0)))) return rc;
    // block column A': its diagonal block on the chain stream (the leaf chain starts on it at once), the rows below on bulk
    if ((rc = upd(wsX, K2, 0, 0, W1, W1, A + ke * lda + ke, 1, side))) return rc;
    if ((rc = upd(wsX, K2, W1, 0, R - ke1, W1, A + ke1 * lda + ke, 0, bulk))) return rc;
    // block column B' (rows from ke1 on): pair update now, on bulk -- ordered before the A' update of the same block below
    if ((rc = upd(wsX, K2, W1, W1, R - ke1, W2, A + ke1 * lda + ke1, 1, bulk))) return rc;
    if ((rc = factor(ke, ke1))) return rc;
    if (W2 > 0) {
      if ((rc = oz_slice_panel(A + ke1 * lda + ke, lda, R - ke1, W1, wsY, R, S, side))) return rc;
      if ((rc = upd(wsY, W1, 0, 0, W2, W2, A + ke1 * lda + ke1, 1, side))) return rc;
      if ((rc = cuda_rc(cudaEventRecord(la.crit, side)))) return rc;  // Y is ready (and every earlier update of B' is done)
      if ((rc = cuda_rc(cudaStreamWaitEvent(bulk, la.crit, 0)))) return rc;
      if ((rc = upd(wsY, W1, W2, 0, R - ke2, W2, A + ke2 * lda + ke1, 0, bulk))) return rc;
      if ((rc = factor(ke1, ke2))) return rc;
    }
    if ((rc = cuda_rc(cudaEventRecord(la.join, side)))) return rc;
    // the far part: everything right of the next pair, K = 1024, on the caller's stream
    if ((rc = upd(wsX, K2, ke2 - ke, ke2 - ke, R - ke2, n_pad - ke2, A + ke2 * lda + ke2, 1, stream))) return rc;
    if ((rc = cuda_rc(cudaStreamWaitEvent(stream, la.join, 0)))) return rc;
  }
  return 0;
}

template <typename T>
static int potrf_driver(T* A, int64_t lda, int64_t a_bs, int64_t n_pad, int64_t extra_rows, T* logdet, int32_t* info,
                        int32_t batch, cudaStream_t stream, Trailing tr = Trailing()) {
  if (!A || n_pad < 0 || extra_rows < 0 || batch < 1 || !info) return GPK_ERR_ARG;
  if (n_pad % NB || extra_rows % NB || lda < n_pad) return GPK_ERR_ARG;
  if (lda % (16 / sizeof(T)) || reinterpret_cast<uintptr_t>(A) % 16) return GPK_ERR_ALIGN;
  const int64_t R = n_pad + extra_rows;
  tr.cap_rows = R;
  int rc;
  Lookahead& la = lookahead();
  if (tr.mode == MODE_OZAKI && sizeof(T) == 8 && batch == 1 && la.ok && n_pad >= 4096 &&
      tr.ws_bytes >= potrf_pairs_ws_bytes(R, tr.slices))
    return potrf_driver_pairs(reinterpret_cast<double*>(A), lda, n_pad, extra_rows, reinterpret_cast<double*>(logdet), info,
                              stream, tr.ws, tr.slices, la);
  const bool use_la = la.ok && n_pad > 2 * NB_OUTER && !no_lookahead();

  const int64_t ke0 = NB_OUTER < n_pad ? NB_OUTER : n_pad;
  if ((rc = factor_panel<T>(A, lda, a_bs, R, 0, ke0, logdet, info, batch, stream))) return rc;
  for (int64_t kb = 0; kb + NB_OUTER < n_pad; kb += NB_OUTER) {
    const int64_t ke = kb + NB_OUTER;                                   // panel [kb, ke) is factorised
    const int64_t ke2 = (ke + NB_OUTER < n_pad) ? ke + NB_OUTER : n_pad;  // next panel [ke, ke2)
    const int64_t K = ke - kb;
    const T* P = A + ke * lda + kb;
    // reduced-cost arithmetic for the trailing update: workspace copy (fp32 / int8 slices) of the panel rows [ke, R)
    int used = MODE_F64;
    if ((rc = prepare_panel<T>(tr, P, lda, R - ke, K, batch, stream, &used))) return rc;
    const bool more = ke2 < n_pad;
    const int64_t W = ke2 - ke;  // width of the next panel
    T* Ckk = A + ke * lda + ke;  // top-left corner of the trailing matrix
    const T* P2 = A + ke2 * lda + kb;
    if (use_la && more) {
      // side streams (high priority): (a) the next panel's columns, then that panel's factorisation;
      // caller's stream: (b) everything to the right of it.  (a) and (b) are independent (both only read panel i), so
      // they run concurrently and the short (a) no longer costs a kernel tail of its own.
      if ((rc = cuda_rc(cudaEventRecord(la.fork, stream)))) return rc;
      if ((rc = cuda_rc(cudaStreamWaitEvent(la.side, la.fork, 0)))) return rc;
      if (used != MODE_TF32X3) {
        // (a) in two parts: the next panel's diagonal block first (the chain starts on it at once), the rows below on `bulk`
        if ((rc = cuda_rc(cudaStreamWaitEvent(la.bulk, la.fork, 0)))) return rc;
        if ((rc = trailing_update<T>(used, tr, 0, 0, W, W, K, P, P, lda, a_bs, Ckk, 1, batch, la.side))) return rc;
        if (R - ke2 > 0 && (rc = trailing_update<T>(used, tr, W, 0, R - ke2, W, K, P2, P, lda, a_bs, A + ke2 * lda + ke, 0,
                                                    batch, la.bulk)))
          return rc;
      } else {
        if ((rc = trailing_update<T>(used, tr, 0, 0, R - ke, W, K, P, P, lda, a_bs, Ckk, 1, batch, la.side))) return rc;
        if ((rc = cuda_rc(cudaStreamWaitEvent(la.bulk, la.fork, 0)))) return rc;
      }
      if ((rc = factor_panel_split<T>(A, lda, a_bs, R, ke, ke2, logdet, info, batch, la.side, la))) return rc;
      if ((rc = cuda_rc(cudaEventRecord(la.join, la.side)))) return rc;
      if ((rc = trailing_update<T>(used, tr, W, W, R - ke2, n_pad - ke2, K, P2, P2, lda, a_bs, A + ke2 * lda + ke2, 1, batch,
                                   stream)))
        return rc;
      if ((rc = cuda_rc(cudaStreamWaitEvent(stream, la.join, 0)))) return rc;
    } else {
      if ((rc = trailing_update<T>(used, tr, 0, 0, R - ke, W, K, P, P, lda, a_bs, Ckk, 1, batch, stream))) return rc;
      if (more) {
        if ((rc = trailing_update<T>(used, tr, W, W, R - ke2, n_pad - ke2, K, P2, P2, lda, a_bs, A + ke2 * lda + ke2, 1,
                                     batch, stream)))
          return rc;
      }
      if ((rc = factor_panel<T>(A, lda, a_bs, R, ke, ke2, logdet, info, batch, stream))) return rc;
    }
  }
  return 0;
}

// X L^T = B, recursive halving (all sizes multiples of 128): the first h columns, the GEMM, then the last n - h columns.
static inline int64_t trsm_split(int64_t n) { return ((n / NB) / 2) * NB; }

template <typename T>
static int trsm_right_rec(const T* L, int64_t ldl, int64_t l_bs, int64_t n, T* B, int64_t ldb, int64_t b_bs,
                          int64_t rows, int32_t batch, int32_t S, void* ws, int64_t ws_bytes, cudaStream_t stream) {
  if (n <= 0) return 0;
  if (n == NB) return trsm_leaf_fwd<T>(L, ldl, l_bs, B, ldb, b_bs, rows, batch, stream);
  const int64_t h = trsm_split(n);
  int rc;
  if ((rc = trsm_right_rec<T>(L, ldl, l_bs, h, B, ldb, b_bs, rows, batch, S, ws, ws_bytes, stream))) return rc;
  if ((rc = gemm_nt(rows, n - h, h, T(-1), B, ldb, b_bs, L + h * ldl, ldl, l_bs, T(1), B + h, ldb, b_bs, 0, batch, S, ws,
                    ws_bytes, stream)))
    return rc;
  return trsm_right_rec<T>(L + h * ldl + h, ldl, l_bs, n - h, B + h, ldb, b_bs, rows, batch, S, ws, ws_bytes, stream);
}

template <typename T>
static int trsm_right_driver(const T* L, int64_t ldl, int64_t l_bs, int64_t n_pad, T* B, int64_t ldb, int64_t b_bs,
                             int64_t rows, int32_t batch, int32_t S, void* ws, int64_t ws_bytes, cudaStream_t stream) {
  if (!L || !B || n_pad < 0 || rows < 0 || batch < 1) return GPK_ERR_ARG;
  if (n_pad % NB || rows % NB || ldl < n_pad || ldb < n_pad) return GPK_ERR_ARG;
  if (ldl % (16 / sizeof(T)) || ldb % (16 / sizeof(T))) return GPK_ERR_ALIGN;
  if ((reinterpret_cast<uintptr_t>(L) | reinterpret_cast<uintptr_t>(B)) % 16) return GPK_ERR_ALIGN;
  if (const int rc = oz_check_emulation(S, ws)) return rc;
  if (rows == 0) return 0;
  return trsm_right_rec<T>(L, ldl, l_bs, n_pad, B, ldb, b_bs, rows, batch, S, ws, ws_bytes, stream);
}

int trsm_right(const double* L, int64_t ldl, int64_t n_pad, double* B, int64_t ldb, int64_t rows, int32_t S, void* ws,
               int64_t ws_bytes, cudaStream_t stream) {
  return trsm_right_driver<double>(L, ldl, 0, n_pad, B, ldb, 0, rows, 1, S, ws, ws_bytes, stream);
}
int trsm_right(const float* L, int64_t ldl, int64_t n_pad, float* B, int64_t ldb, int64_t rows, int32_t, void*, int64_t,
               cudaStream_t stream) {
  return trsm_right_driver<float>(L, ldl, 0, n_pad, B, ldb, 0, rows, 1, 0, nullptr, 0, stream);
}

// X L = B (backward substitution), right-looking over 128-blocks from the last to the first.  The off-diagonal
// update  B[:, 0:j] -= X_j L[j, 0:j]  is a rank-128 "NN" product; it is expressed with gemm_nt through an explicit
// transposed copy of the L row-panel made by the caller-provided scratch -- used only for few right-hand sides
// (autograd, sparse mu), so the simple blocked form is enough.
template <typename T>
__global__ void trsm_t_update_kernel(const T* __restrict__ L, int64_t ldl, int64_t l_bs, T* __restrict__ B,
                                     int64_t ldb, int64_t b_bs, int64_t j0, int64_t rows) {
  // B[r][c] -= sum_{q < 128} B[r][j0 + q] * L[j0 + q][c]   for c < j0 ; one thread per (r, c)
  const int bidx = blockIdx.z;
  L += (int64_t)bidx * l_bs;
  B += (int64_t)bidx * b_bs;
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t r = blockIdx.y;
  __shared__ T xs[NB];
  if (threadIdx.x < NB) xs[threadIdx.x] = B[r * ldb + j0 + threadIdx.x];
  __syncthreads();
  if (c >= j0 || r >= rows) return;
  T s = T(0);
#pragma unroll 8
  for (int q = 0; q < NB; ++q) s = fma(xs[q], L[(j0 + q) * ldl + c], s);
  B[r * ldb + c] -= s;
}

template <typename T>
static int trsm_right_t_driver(const T* L, int64_t ldl, int64_t l_bs, int64_t n_pad, T* B, int64_t ldb, int64_t b_bs,
                               int64_t rows, int32_t batch, cudaStream_t stream) {
  if (!L || !B || n_pad < 0 || rows < 0 || batch < 1) return GPK_ERR_ARG;
  if (n_pad % NB || rows % 64 || ldl < n_pad || ldb < n_pad) return GPK_ERR_ARG;
  if (rows == 0) return 0;
  int rc;
  for (int64_t j = n_pad - NB; j >= 0; j -= NB) {
    if ((rc = launch_trsm_leaf<T>(L + j * ldl + j, ldl, l_bs, B + j, ldb, b_bs, rows, batch, stream))) return rc;
    if (j > 0) {
      dim3 grid((unsigned)((j + 127) / 128), (unsigned)rows, (unsigned)batch);
      trsm_t_update_kernel<T><<<grid, 128, 0, stream>>>(L, ldl, l_bs, B, ldb, b_bs, j, rows);
      GPK_COUNT_LAUNCH();
      GPK_CHECK_LAUNCH();
    }
  }
  return 0;
}

}  // namespace gpk

extern "C" {
int gpk_debug_leaf_phase_clock(void* buf16_int64) {
  long long* p = static_cast<long long*>(buf16_int64);
  return gpk::cuda_rc(cudaMemcpyToSymbol(gpk::g_leaf_phase_clock, &p, sizeof(p)));
}
int64_t gpk_potrf_oz_ws_bytes(int64_t n_pad, int64_t extra_rows, int32_t slices) {
  if (slices < 5 || slices > 8 || n_pad < 2048) return 0;
  const int64_t one = gpk::oz_ws_bytes(n_pad + extra_rows, gpk::NB_OUTER, slices);
  const int64_t pairs = gpk::potrf_pairs_ws_bytes(n_pad + extra_rows, slices);  // the pair scheme (n_pad >= 4096)
  return n_pad >= 4096 && pairs > one ? pairs : one;
}
int64_t gpk_trsm_right_oz_ws_bytes(int64_t n_pad, int64_t rows, int32_t slices) {
  if (n_pad <= gpk::NB) return 0;
  const int64_t h = gpk::trsm_split(n_pad);
  int64_t need = gpk_gemm_nt_oz_ws_bytes(rows, n_pad - h, h, slices);
  for (const int64_t part : {gpk_trsm_right_oz_ws_bytes(h, rows, slices), gpk_trsm_right_oz_ws_bytes(n_pad - h, rows, slices)})
    need = part > need ? part : need;
  return need;
}
int gpk_potrf_f64(double* A, int64_t lda, int64_t a_bstride, int64_t n_pad, int64_t extra_rows, double* logdet,
                  int32_t* info, int32_t batch, int32_t slices, void* ws, int64_t ws_bytes, void* stream) {
  if (const int rc = gpk::oz_check_emulation(slices, ws)) return rc;
  gpk::Trailing t;
  // the int8-slice emulation of the trailing updates: one large matrix, and the scratch holds a panel's slices
  if (slices && batch == 1 && n_pad >= 2048 && ws_bytes >= gpk::oz_ws_bytes(n_pad + extra_rows, gpk::NB_OUTER, slices)) {
    t.mode = gpk::MODE_OZAKI;
    t.ws = ws;
    t.ws_bytes = ws_bytes;
    t.slices = slices;
  }
  return gpk::potrf_driver<double>(A, lda, a_bstride, n_pad, extra_rows, logdet, info, batch, (cudaStream_t)stream, t);
}
int gpk_potrf_f64_tf32x3(double* A, int64_t lda, int64_t a_bstride, int64_t n_pad, int64_t extra_rows, double* logdet,
                         int32_t* info, int32_t batch, float* ws, int64_t ws_elems, void* stream) {
  gpk::Trailing t;
  t.mode = gpk::MODE_TF32X3;
  t.ws = ws;
  t.ws_bytes = ws_elems * 4;
  return gpk::potrf_driver<double>(A, lda, a_bstride, n_pad, extra_rows, logdet, info, batch, (cudaStream_t)stream, t);
}
int gpk_potrf_f32(float* A, int64_t lda, int64_t a_bstride, int64_t n_pad, int64_t extra_rows, float* logdet,
                  int32_t* info, int32_t batch, void* stream) {
  return gpk::potrf_driver<float>(A, lda, a_bstride, n_pad, extra_rows, logdet, info, batch, (cudaStream_t)stream);
}
int gpk_trsm_right_f64(const double* L, int64_t ldl, int64_t l_bstride, int64_t n_pad, double* B, int64_t ldb,
                       int64_t b_bstride, int64_t rows, int32_t batch, int32_t slices, void* ws, int64_t ws_bytes,
                       void* stream) {
  return gpk::trsm_right_driver<double>(L, ldl, l_bstride, n_pad, B, ldb, b_bstride, rows, batch, slices, ws, ws_bytes,
                                        (cudaStream_t)stream);
}
int gpk_trsm_right_f32(const float* L, int64_t ldl, int64_t l_bstride, int64_t n_pad, float* B, int64_t ldb,
                       int64_t b_bstride, int64_t rows, int32_t batch, void* stream) {
  return gpk::trsm_right_driver<float>(L, ldl, l_bstride, n_pad, B, ldb, b_bstride, rows, batch, 0, nullptr, 0,
                                       (cudaStream_t)stream);
}
int gpk_trsm_right_t_f64(const double* L, int64_t ldl, int64_t l_bstride, int64_t n_pad, double* B, int64_t ldb,
                         int64_t b_bstride, int64_t rows, int32_t batch, void* stream) {
  return gpk::trsm_right_t_driver<double>(L, ldl, l_bstride, n_pad, B, ldb, b_bstride, rows, batch,
                                          (cudaStream_t)stream);
}
int gpk_trsm_right_t_f32(const float* L, int64_t ldl, int64_t l_bstride, int64_t n_pad, float* B, int64_t ldb,
                         int64_t b_bstride, int64_t rows, int32_t batch, void* stream) {
  return gpk::trsm_right_t_driver<float>(L, ldl, l_bstride, n_pad, B, ldb, b_bstride, rows, batch,
                                         (cudaStream_t)stream);
}
}
