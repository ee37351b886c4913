// fp64 GEMM  C = beta*C + alpha * A * B^T  emulated on the Hopper tensor cores' INT8 path (wgmma.mma_async .s32.s8.s8,
// int32 accumulators in registers) with the Ozaki splitting: every row of A and B is scaled by a power of two (its
// largest magnitude) and cut into S signed 7-bit slices
//        a = 2^e * sum_s  q_s 2^-(6+7s),   q_s = round-to-nearest of the running remainder, |q_s| <= 64   (error-free)
// so that   a . b = 2^(e_a+e_b) * sum_{s,t} 2^-(12+7(s+t)) * (q_s . r_t),   and every integer dot product q_s . r_t is
// EXACT in int32 (|q r| <= 2^12, K <= 65536, up to S products per accumulator).  Products with s + t >= S are dropped
// (they are below the slicing error), leaving S(S+1)/2 int8 GEMMs -- 21 for S = 6 (error ~2^-40 of |a||b|, zero-mean), 28
// for S = 7 (~2^-47).
//
// 128 x 64 output tiles, a few consecutive tiles per cluster, enumerated in bands of tile rows, column-major inside a band
// (tiles in flight share the band's A slices in L2; oz_tile).  Products with the same s + t share an accumulator, so a tile
// needs S int32 accumulators per element: 128 x 64 x S does not fit the registers of two warpgroups, so every tile is
// computed as two halves of 128 x 32 (S x 16 accumulator registers per thread, 128 for S = 8), side by side by the two
// CTAs of a cluster: CTA rank r computes columns 32 r .. 32 r + 31 of every tile of its cluster.  Both need all 128 A rows,
// so each loads one 64-row half of A and multicasts it into both: a tile reads its A slices from L2 once, not twice.
//   warpgroup 0   TMA producer (one thread): per 64-byte k-block ONE box {64 B, 64 rows, S slices} of A (rows 64 r ..,
//                 multicast to both CTAs of the cluster) and one {64 B, 32 rows, S} of B (this CTA's columns)
//                 (cp.async.bulk.tensor.3d, SWIZZLE_64B, mbarrier complete_tx) into a ring.  A stage is laid out
//                 [A row half][S][64 rows][64 B], then B; it is refilled once the consumers of BOTH CTAs released it
//   warpgroups 1-2  consumers, rows 0-63 / 64-127 of the tile: per K = 32 step, slice s of A against slices 0..S-1-s of B,
//                 grouped by PAIRS of diagonals {0,1}, {2,3}, ... (B slices adjacent in shared memory, accumulators
//                 adjacent in the register fragment): for each group {lo, lo+1} with lo > s - 1 one wgmma with N = 64 (32
//                 for a last, single diagonal) over B slices lo - s, lo - s + 1.  For odd s diagonal s alone is left: at
//                 S <= 7 it goes to an extra accumulator (16 registers, folded into diagonal s by an exact int32 add
//                 before the epilogue), at S = 8 (no registers for 4 extras) the group {s-1, s} runs over a zero B block
//                 placed in front of B slice 0.  So every wgmma writes a whole group or an extra accumulator: runs that
//                 partially overlap would make ptxas serialise the chain, one wgmma in flight at a time.  All wgmmas of a
//                 64-byte k-block are issued in one go (19 per K = 32 step at S = 7, 20 at S = 8) with A from registers
//                 (ldmatrix from the swizzled stage) for as many slices as the register budget allows, the rest from
//                 shared memory.  Then the epilogue: Horner-combine the S diagonals in fp64 (exact int32 -> double
//                 through the 2^52 trick), scale by 2^(e_row + e_col) and add into C (red.global.add.f64: the
//                 read-modify-write happens in L2, as one correctly rounded addition per element)
// Rows of every finite magnitude (subnormal to near overflow) are scaled exactly, and the exponents are summed as integers
// before the scale is applied, so products of very small rows with very large ones keep the full accuracy.  A row with a
// NaN or an infinity makes its whole row (column) of the product NaN -- where fp64 gives NaN or +-inf.
// The slicing kernel (oz_slice_kernel) is O(rows*K) and runs once per panel; in the Cholesky its output is shared by
// every tile of the trailing update.  Every inexact step is ONE correctly rounded fp64 operation, so the result equals a
// NumPy integer model of the algorithm bit for bit (tests/_oz_model.py, tests/test_emulation.py).
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace gpk {
namespace {

constexpr int OZ_BM = 128, OZ_BN = 64, OZ_BK = 64;  // BK in bytes = int8 elements
constexpr int OZ_HN = 32;                           // columns per pass (half a tile)
constexpr int OZ_THREADS = 384;

template <int S>
struct OzCfg {
  // Diagonal schedule (see the header): PAD = zero block in front of B slice 0 (odd A slices use a window starting in it),
  // otherwise odd diagonals get EXTRA accumulators of their own.  The first RA A slices are read into registers (8 per
  // slice and k-block), the rest straight from shared memory, so that accumulators + A fragments stay within 192 of the
  // consumers' 232 registers: S <= 6 all in registers; S = 7: 160 accumulators, slices 0-3 in registers; S = 8 would need
  // 192 accumulators, so it pads (3 resp. 4 zero products per K = 32 step on top of 28 resp. 36 for S = 7 / 8 padded) and
  // keeps its 8 slices in registers.
  static constexpr bool PAD = S > 7;
  static constexpr int EXTRA = PAD ? 0 : S / 2;
  static constexpr int ACC = 16 * (S + EXTRA);  // int32 accumulator registers per thread
  static constexpr int RA = (192 - ACC) / 8 < S ? (192 - ACC) / 8 : S;
  static constexpr int A_SLICE = 64 * OZ_BK;     // 4 KB: one 64-row half of an A slice
  static constexpr int A_HALF = S * A_SLICE;     // a row half, all slices: one multicast box, one consumer warpgroup's rows
  static constexpr int B_SLICE = OZ_HN * OZ_BK;  // 2 KB
  static constexpr int A_BYTES = 2 * A_HALF;
  static constexpr int Z_BYTES = PAD ? B_SLICE : 0;
  static constexpr int B_BYTES = S * B_SLICE;
  static constexpr int TX_BYTES = A_BYTES + B_BYTES;  // what the TMA writes per stage: both A halves (own + peer) and B
  static constexpr int STAGE_BYTES = A_BYTES + Z_BYTES + B_BYTES;
  static constexpr int SMEM_MAX = 226 * 1024;  // 227 KB per CTA minus the static barriers / alignment slack
  static constexpr int STAGES = (SMEM_MAX - 1024) / STAGE_BYTES > 4 ? 4 : (SMEM_MAX - 1024) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024;
  static_assert(STAGES >= 2, "ring");
};

// Row exponent of a row holding a NaN or an infinity: every element of the product that the row touches becomes NaN
constexpr int32_t OZ_E_NONFINITE = 1 << 20;

// 2^e for e in [-1022, 1023] (a normal double)
__device__ __forceinline__ double oz_pow2(int e) { return __hiloint2double((1023 + e) << 20, 0); }

// x 2^E for E outside the normal range: two normal powers of two, the larger one first (x 2^-1022 stays exact for |x| >= 1,
// so only the last product rounds); NaN for the exponent of a non-finite row
__device__ __forceinline__ double oz_scale_wide(double x, int E) {
  if (E > OZ_E_NONFINITE / 2) return __longlong_as_double(0x7ff8000000000000ll);
  const int e1 = E < 0 ? -1022 : 1023;
  return x * oz_pow2(e1) * oz_pow2(max(E - e1, -1022));
}

struct OzParams {
  double alpha;
  double* C;
  const int32_t* ex_a;  // row exponent e per A row (already offset to the first row of the problem)
  const int32_t* ex_b;
  int64_t ldc;
  int32_t a_row0, b_row0;  // first plane row of A / B
  int32_t KB, lower, tiles_m, tiles_n;
  int32_t total_tiles, tiles_per_cta, tri_rows;  // tri_rows: tile rows in the triangular part (lower mode)
  int32_t accumulate;                            // 1: C += alpha A B^T (reduce-add), 0: C = alpha A B^T (store)
  int32_t band;                                  // tile rows per band of the tile order
};

__device__ __forceinline__ void oz_mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "OZW_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra OZW_DONE;\n"
      "bra OZW_LOOP;\n"
      "OZW_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// the producer's wait for a free stage: the releases come from the consumers of both CTAs (mbar_arrive_cluster)
__device__ __forceinline__ void oz_mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "OZC_LOOP:\n"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra OZC_DONE;\n"
      "bra OZC_LOOP;\n"
      "OZC_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void oz_tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}
// exact int32 -> double without the conversion pipe: bits(2^52 + 2^31 + x) = 0x43300000 : (x ^ 0x80000000)
__device__ __forceinline__ double oz_i2d(uint32_t x) {
  return __hiloint2double(0x43300000, (int)(x ^ 0x80000000u)) - 4503601774854144.0;  // 2^52 + 2^31
}
// A slice SA (64 rows) times the N rows of B at b_addr: A from its registers a + 4 SA (SA < RA) or from the stage (a_addr)
template <int S, int SA, int N>
__device__ __forceinline__ void oz_wgmma(uint32_t* d, const uint32_t* a, uint32_t a_addr, uint32_t b_addr, uint32_t accumulate) {
  if constexpr (SA < OzCfg<S>::RA)
    wgmma_s8_ra<N>(d, a + 4 * SA, wgmma_desc<64>(b_addr), accumulate);
  else
    wgmma_s8<N>(d, wgmma_desc<64>(a_addr + SA * OzCfg<S>::A_SLICE), wgmma_desc<64>(b_addr), accumulate);
}
// Diagonal group {LO, LO + 1} (or the last, single {S - 1}) of A slice SA: B slices LO - SA .. into accumulators LO ..
template <int S, int SA, int LO>
__device__ __forceinline__ void oz_mma_groups(uint32_t* acc, const uint32_t* a, uint32_t a_addr, uint32_t b_addr,
                                              uint32_t accumulate) {
  constexpr int W = S - LO < 2 ? S - LO : 2;
  oz_wgmma<S, SA, OZ_HN * W>(acc + 16 * LO, a, a_addr, b_addr + (LO - SA) * OzCfg<S>::B_SLICE, accumulate);
  if constexpr (LO + 2 < S) oz_mma_groups<S, SA, LO + 2>(acc, a, a_addr, b_addr, accumulate);
}
// One K = 32 step of a consumer warpgroup: A slice SA against B slices 0 .. S-1-SA.  Every wgmma writes a whole diagonal
// group or an extra accumulator, so no two of them write overlapping, unequal register runs (which makes ptxas serialise
// the wgmma chain).  The first step of a pass (accumulate = 0) starts with SA = 0, which writes every group.
template <int S, int SA>
__device__ __forceinline__ void oz_mma_step(uint32_t* acc, const uint32_t* a, uint32_t a_addr, uint32_t b_addr,
                                            uint32_t accumulate) {
  using Cfg = OzCfg<S>;
  if constexpr (SA & 1) {
    if constexpr (Cfg::PAD)  // group {SA - 1, SA}: window from the zero block in front of B slice 0
      oz_wgmma<S, SA, 2 * OZ_HN>(acc + 16 * (SA - 1), a, a_addr, b_addr - Cfg::B_SLICE, 1u);
    else  // diagonal SA alone, into its extra accumulator
      oz_wgmma<S, SA, OZ_HN>(acc + 16 * (S + SA / 2), a, a_addr, b_addr, accumulate);
  }
  constexpr int LO = (SA + 1) & ~1;  // first group that lies wholly at or above diagonal SA
  if constexpr (LO < S) oz_mma_groups<S, SA, LO>(acc, a, a_addr, b_addr, SA == 0 ? accumulate : 1u);
  if constexpr (SA + 1 < S) oz_mma_step<S, SA + 1>(acc, a, a_addr, b_addr, accumulate);
}
// tile index -> (tile row, tile column).  Lower mode enumerates only the tiles that touch the lower triangle: row tm holds
// nc(tm) = min(tiles_n, 2 (tm + 1)) tiles (128 x 64 tiles), so f(r) = r (r + 1) tiles precede row r while r <= tri_rows.
// Order: BANDS of `band` (16) tile rows, column-major inside a band.  Tiles that run at the same time then share the band's A rows
// (16 x 128 rows of slices: 15 MB at K = 1024, S = 7) and sweep the B rows once per band, instead of once per tile ROW
// as the plain row-major order did -- whose K = 1024 launches read 2.1x their algorithmic bytes from HBM (ncu, round 2: the
// 104 MB of slices no longer fit L2 next to the C traffic).
__host__ __device__ __forceinline__ int oz_rows_before(const OzParams& p, int r) {  // tiles in tile rows < r
  if (!p.lower) return r * p.tiles_n;
  return r <= p.tri_rows ? r * (r + 1) : p.tri_rows * (p.tri_rows + 1) + (r - p.tri_rows) * p.tiles_n;
}
__host__ __device__ __forceinline__ void oz_tile(const OzParams& p, int t, int& tm, int& tn) {
  // (1) band
  int r0 = 0;
  while (r0 + p.band < p.tiles_m && oz_rows_before(p, r0 + p.band) <= t) r0 += p.band;
  const int r1 = (r0 + p.band < p.tiles_m) ? r0 + p.band : p.tiles_m;
  int u = t - oz_rows_before(p, r0);
  // (2) column-major inside the band: row tm has nc(tm) columns, non-decreasing in tm
  const int nc0 = (p.lower && 2 * (r0 + 1) < p.tiles_n) ? 2 * (r0 + 1) : p.tiles_n;  // columns that every row of the band has
  const int h = r1 - r0;
  if (u < nc0 * h) {
    tn = u / h;
    tm = r0 + (u - tn * h);
    return;
  }
  u -= nc0 * h;
  // ragged part (lower mode only): column c >= nc0 exists in the rows tm with 2 (tm + 1) > c, i.e. tm = c / 2 ... r1 - 1
  for (int c = nc0; c < p.tiles_n; ++c) {
    const int first = (c >> 1) > r0 ? (c >> 1) : r0;  // first row of the band that has column c (c < tiles_n is implied by u's range)
    const int cnt = r1 - first;
    if (u < cnt) {
      tn = c;
      tm = first + u;
      return;
    }
    u -= cnt;
  }
  tm = r1 - 1;  // not reached for t < total_tiles (bijection checked on the host for 1047 shapes); keeps the loop bounded
  tn = p.tiles_n - 1;
}

// Launched as clusters of 2 CTAs (oz_launch_gemm).  A cluster works through `tiles_per_cta` consecutive tiles; CTA rank r
// computes the 128 x 32 half r of each.  The TMA producer runs ahead through the ring into the next tile while the
// consumers finish the current one.  Both CTAs walk the same tiles and k-blocks, so their rings stay in step.  Clusters
// stay short-lived (a few tiles) on purpose: the Cholesky's look-ahead stream needs SMs to come free every few tens of us.
template <int S>
__global__ void __launch_bounds__(OZ_THREADS, 1)
oz_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const OzParams p) {
  using Cfg = OzCfg<S>;
  constexpr int STAGES = Cfg::STAGES;
  const int wg = threadIdx.x >> 7;
  const uint32_t rank = cluster_ctarank();  // A row half this CTA loads for both, column half of every tile it computes
  const int t_begin = (blockIdx.x >> 1) * p.tiles_per_cta;
  const int t_end = min(t_begin + p.tiles_per_cta, p.total_tiles);

  extern __shared__ uint8_t oz_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(oz_smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);  // this CTA's producer (expect_tx of both A halves and B)
      mbar_init(&empty_bar[s], 2 * 8);  // lane 0 of each of the 8 consumer warps of BOTH CTAs, after its MMAs on the stage
    }
    fence_mbar_init();
  }
  if constexpr (Cfg::PAD) {  // the zero blocks: written once, never touched by the TMA, read by the wgmmas (async proxy)
    for (int i = threadIdx.x; i < STAGES * Cfg::Z_BYTES / 16; i += OZ_THREADS) {
      const int st = i / (Cfg::Z_BYTES / 16), j = i % (Cfg::Z_BYTES / 16);
      reinterpret_cast<uint4*>(smem + st * Cfg::STAGE_BYTES + Cfg::A_BYTES)[j] = make_uint4(0, 0, 0, 0);
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
  }
  cluster_sync();  // no multicast or remote arrive may reach the peer's barriers before it initialised them
  const int KB = p.KB;

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::);
    if (threadIdx.x == 0) {
      int g = 0;  // k-blocks issued so far (all tiles)
      for (int t = t_begin; t < t_end; ++t) {
        int tm, tn;
        oz_tile(p, t, tm, tn);
        for (int kb = 0; kb < KB; ++kb, ++g) {
          const int s = g % STAGES, it = g / STAGES;
          if (it > 0) oz_mbar_wait_cluster(&empty_bar[s], (it - 1) & 1);  // both CTAs done with the stage's last use
          uint8_t* st = smem + s * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[s], Cfg::TX_BYTES);
          tma_load_3d_multicast(st + rank * Cfg::A_HALF, &mapA, kb * OZ_BK, p.a_row0 + tm * OZ_BM + 64 * rank, 0,
                                &full_bar[s], 0x3);
          oz_tma_load_3d(st + Cfg::A_BYTES + Cfg::Z_BYTES, &mapB, kb * OZ_BK, p.b_row0 + tn * OZ_BN + rank * OZ_HN, 0,
                         &full_bar[s]);
        }
      }
      // before this CTA may exit: the last use of every stage released by the consumers of BOTH CTAs, i.e. every remote
      // arrive on our barriers has landed (every multicast into our stages has, since our consumers waited for them).
      // Cheaper than a cluster barrier with release semantics, whose MEMBAR.GPU waits for the epilogue's reductions
      for (int u = g > STAGES ? g - STAGES : 0; u < g; ++u) oz_mbar_wait_cluster(&empty_bar[u % STAGES], (u / STAGES) & 1);
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::);
    const int tid = threadIdx.x - 128 * wg, half = wg - 1;  // thread in the warpgroup, the A row half (64 rows) it owns
    const int r_lo = 16 * (tid >> 5) + ((tid & 31) >> 2), c_lo = 2 * (tid & 3);
    // ldmatrix.x4 source of this lane inside its row half of an A slice, for the two K = 32 halves of the 64-byte
    // (SWIZZLE_64B) row: matrix lane / 8 = rows +8 (bit 0) and bytes +16 (bit 1), 16-byte chunk XOR (row / 2) % 4
    const int lane = tid & 31, a_row = 16 * (tid >> 5) + (lane & 7) + 8 * ((lane >> 3) & 1);
    const uint32_t a_off0 = half * Cfg::A_HALF + a_row * OZ_BK + ((((lane >> 4) + 0) ^ ((lane >> 1) & 3)) << 4);
    const uint32_t a_off1 = half * Cfg::A_HALF + a_row * OZ_BK + ((((lane >> 4) + 2) ^ ((lane >> 1) & 3)) << 4);
    uint32_t acc[Cfg::ACC];
    int g = 0;
    for (int t = t_begin; t < t_end; ++t) {
      int tm, tn;
      oz_tile(p, t, tm, tn);
      // ---- main loop: all wgmmas of a k-block in flight at once, A fragments in registers ----
      for (int kb = 0; kb < KB; ++kb, ++g) {
        const int s = g % STAGES, it = g / STAGES;
        oz_mbar_wait(&full_bar[s], it & 1);
        const uint32_t st = smem_u32(smem + s * Cfg::STAGE_BYTES), b0 = st + Cfg::A_BYTES + Cfg::Z_BYTES;
        uint32_t a[2][4 * Cfg::RA];
#pragma unroll
        for (int sl = 0; sl < Cfg::RA; ++sl) {
          ldmatrix_x4(a[0] + 4 * sl, st + sl * Cfg::A_SLICE + a_off0);
          ldmatrix_x4(a[1] + 4 * sl, st + sl * Cfg::A_SLICE + a_off1);
        }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 2; ++ks)  // wgmma K = 32 int8 = 32 bytes inside the 64-byte swizzle row
          oz_mma_step<S, 0>(acc, a[ks], st + half * Cfg::A_HALF + ks * 32, b0 + ks * 32, (kb > 0 || ks > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();  // (the A registers are rewritten by the next k-block; the other consumer keeps the tensor cores busy)
        if (lane == 0) {  // the stage is free for this warp in both CTAs (the peer multicasts its A half into ours)
          mbar_arrive_cluster(&empty_bar[s], 0);
          mbar_arrive_cluster(&empty_bar[s], 1);
        }
      }
      // ---- epilogue: Horner-combine the diagonals in fp64, scale, add into C ----
      if constexpr (Cfg::EXTRA > 0) {  // fold the extra accumulators into their diagonals (exact int32 sums)
#pragma unroll
        for (int d = 1; d < S; d += 2)
#pragma unroll
          for (int i = 0; i < 16; ++i) acc[16 * d + i] += acc[16 * (S + d / 2) + i];
      }
      const int64_t row0 = (int64_t)tm * OZ_BM + 64 * half + r_lo;
      const int64_t col0 = (int64_t)tn * OZ_BN + rank * OZ_HN + c_lo;
      // Scaling: out = v alpha 2^E, E = e_row + e_col - W (W: the weight of the last kept diagonal; Horner ran from
      // diagonal 0 down), rounded once.  This thread's 2 rows and 8 columns give factors ra = alpha 2^(e_row - W) and
      // cb = 2^e_col.  When all of them and all their products are normal doubles (the usual case), ra cb = alpha 2^E
      // exactly and out = v (ra cb) is that one rounding.  Otherwise (rows far from 1, non-finite rows) E is summed as
      // an integer per element and applied last to v alpha, in two power-of-two factors when it lies outside the normal
      // range: one rounding for every normal result, and nothing goes subnormal before the result does
      constexpr int W = 12 + 7 * (S - 1);
      double ra[2], cb[8];
      bool fast = true;
      double ra_min = 1.0 / 0.0, ra_max = 0.0;
      int eb_min = 1023, eb_max = -1022;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int e = __ldg(p.ex_a + row0 + 8 * h) - W;
        fast = fast && (unsigned)(e + 1022) <= 2045u;
        ra[h] = p.alpha * oz_pow2(min(max(e, -1022), 1023));
        ra_min = fmin(ra_min, fabs(ra[h]));
        ra_max = fmax(ra_max, fabs(ra[h]));
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int e = __ldg(p.ex_b + col0 + 8 * (q >> 1) + (q & 1));
        fast = fast && (unsigned)(e + 1022) <= 2045u;
        eb_min = min(eb_min, e);
        eb_max = max(eb_max, e);
        cb[q] = oz_pow2(min(max(e, -1022), 1023));
      }
      constexpr double DBL_MIN_NORMAL = 2.2250738585072014e-308;
      fast = fast && ra_min >= DBL_MIN_NORMAL && ra_max <= 1.7976931348623157e308 &&
             ra_min * oz_pow2(max(eb_min, -1022)) >= DBL_MIN_NORMAL &&
             ra_max * oz_pow2(min(eb_max, 1023)) <= 1.7976931348623157e308;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int64_t row = row0 + 8 * ((i >> 1) & 1), col = col0 + 8 * (i >> 2) + (i & 1);
        double v = oz_i2d(acc[i]);
#pragma unroll
        for (int d = 1; d < S; ++d) v = fma(v, 128.0, oz_i2d(acc[16 * d + i]));
        double out;
        if (fast) {
          out = v * (ra[(i >> 1) & 1] * cb[2 * (i >> 2) + (i & 1)]);
        } else {
          const int E = __ldg(p.ex_a + row) + __ldg(p.ex_b + col) - W;
          out = v * p.alpha;
          if ((unsigned)(E + 1022) <= 2045u)
            out *= oz_pow2(E);
          else
            out = oz_scale_wide(out, E);
        }
        double* c = p.C + row * p.ldc + col;
        if (p.accumulate)
          atomicAdd(c, out);
        else
          *c = out;
      }
    }
  }
}

// ---- slicing: one warp per row.  planes[s][row][k] (int8), ex[row] = e -------------------------------------------------
// e = ilogb(row max) + 1 over the whole finite range (subnormal rows included: e in [-1073, 1024]), 0 for an all-zero row.
// A row holding a NaN or an infinity gets e = OZ_E_NONFINITE and zero slices: its row (column) of the product is NaN, as
// it is in fp64 -- and a factorisation then reports the first pivot the non-finite value reaches, as the native path does.
template <int S>
__global__ void __launch_bounds__(256)
oz_slice_kernel(const double* __restrict__ P, int64_t ldp, int64_t rows, int32_t K, int8_t* __restrict__ planes,
                int64_t plane_stride, int32_t* __restrict__ ex) {
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const double* src = P + row * ldp;
  double m = 0.0;
  bool finite = true;
  for (int k = lane * 4; k < K; k += 128) {
    const double2 a = *reinterpret_cast<const double2*>(src + k), b = *reinterpret_cast<const double2*>(src + k + 2);
    m = fmax(fmax(fabs(a.x), fabs(a.y)), fmax(m, fmax(fabs(b.x), fabs(b.y))));
    finite = finite && isfinite(a.x) && isfinite(a.y) && isfinite(b.x) && isfinite(b.y);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  finite = __all_sync(0xffffffffu, finite);
  // r = x 2^-e, as two exact power-of-two scalings (2^-e itself is not a double for e < -1022 or e > 1023)
  int e = 0;
  double inv1 = finite ? 1.0 : 0.0, inv2 = 1.0;
  if (!finite) {
    e = OZ_E_NONFINITE;
  } else if (m > 0.0) {
    e = ilogb(m) + 1;
    const int s1 = min(max(-e, -1022), 1023);
    inv1 = oz_pow2(s1);
    inv2 = oz_pow2(-e - s1);
  }
  if (lane == 0) ex[row] = e;
  int8_t* dst = planes + row * K;
  for (int k = lane * 4; k < K; k += 128) {
    const double2 a = *reinterpret_cast<const double2*>(src + k), b = *reinterpret_cast<const double2*>(src + k + 2);
    double r[4] = {a.x * inv1 * inv2, a.y * inv1 * inv2, b.x * inv1 * inv2, b.y * inv1 * inv2};
    if (!finite) r[0] = r[1] = r[2] = r[3] = 0.0;
    double pw = 64.0, ipw = 1.0 / 64.0;
#pragma unroll
    for (int s = 0; s < S; ++s) {
      char4 q;
      double t;
      t = rint(r[0] * pw); r[0] = fma(-t, ipw, r[0]); q.x = (signed char)(int)t;
      t = rint(r[1] * pw); r[1] = fma(-t, ipw, r[1]); q.y = (signed char)(int)t;
      t = rint(r[2] * pw); r[2] = fma(-t, ipw, r[2]); q.z = (signed char)(int)t;
      t = rint(r[3] * pw); r[3] = fma(-t, ipw, r[3]); q.w = (signed char)(int)t;
      *reinterpret_cast<char4*>(dst + (int64_t)s * plane_stride + k) = q;
      pw *= 128.0;
      ipw *= 1.0 / 128.0;
    }
  }
}

static bool oz_make_map(CUtensorMap* m, const int8_t* planes, int64_t K, int64_t rows_cap, int64_t plane_stride, int S,
                        int box_rows) {
  const EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return false;
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)rows_cap, (cuuint64_t)S};
  cuuint64_t strides[2] = {(cuuint64_t)K, (cuuint64_t)plane_stride};
  cuuint32_t box[3] = {(cuuint32_t)OZ_BK, (cuuint32_t)box_rows, (cuuint32_t)S};
  cuuint32_t es[3] = {1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<int8_t*>(planes), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int S>
int oz_launch_slice(const double* P, int64_t ldp, int64_t rows, int64_t K, int8_t* planes, int64_t plane_stride, int32_t* ex,
                    cudaStream_t stream) {
  if (rows == 0) return 0;
  oz_slice_kernel<S><<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(P, ldp, rows, (int32_t)K, planes, plane_stride, ex);
  GPK_COUNT_LAUNCH();
  return cuda_rc(cudaGetLastError());
}

// C *= beta on the elements the GEMM kernel writes: all of C, or in lower mode the tiles that touch the lower triangle
// (row i: columns below 128 (i / 128 + 1)).  One block per row.
__global__ void oz_scale_kernel(double* C, int64_t ldc, int64_t N, double beta, int32_t lower) {
  const int64_t i = (int64_t)blockIdx.x;
  const int64_t n = lower ? min(N, (i / OZ_BM + 1) * OZ_BM) : N;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) C[i * ldc + j] *= beta;
}

template <int S>
int oz_launch_gemm(int64_t M, int64_t N, int64_t K, double alpha, const int8_t* planesA, int64_t capA, int64_t strideA,
                   const int32_t* exA, int64_t rowA, const int8_t* planesB, int64_t capB, int64_t strideB,
                   const int32_t* exB, int64_t rowB, double beta, double* C, int64_t ldc, int32_t lower,
                   cudaStream_t stream) {
  CUtensorMap mA, mB;
  if (!oz_make_map(&mA, planesA, K, capA, strideA, S, OZ_BM / 2) || !oz_make_map(&mB, planesB, K, capB, strideB, S, OZ_HN))
    return GPK_ERR_UNSUPPORTED;
  if (const int rc = opt_in_smem<oz_gemm_kernel<S>>(OzCfg<S>::SMEM_BYTES)) return rc;
  if (beta != 0.0 && beta != 1.0) {  // the kernel adds into C (or overwrites it): apply any other beta first
    oz_scale_kernel<<<(unsigned)M, 256, 0, stream>>>(C, ldc, N, beta, lower);
    GPK_COUNT_LAUNCH();
  }
  const int32_t tiles_m = (int32_t)(M / OZ_BM), tiles_n = (int32_t)(N / OZ_BN);
  const int32_t tri_rows = lower ? (tiles_m < tiles_n / 2 ? tiles_m : tiles_n / 2) : 0;
  const int32_t total = lower ? tri_rows * (tri_rows + 1) + (tiles_m - tri_rows) * tiles_n : tiles_m * tiles_n;
  // tiles per cluster: >= 2 waves of CTAs (132 clusters of 2) over the H100's 132 SMs before clusters grow, and CTAs stay
  // short-lived (look-ahead streams need SMs every few tens of us): at most 2 tiles at K > 512, 4 below.  At n = 16384
  // (400 W H100) the log-pdf step was 1.7 % slower with caps of 4 / 8, and 8 / 16 was another 3.3 % slower than 4 / 8
  const int32_t tpc_cap = K > 512 ? 2 : 4;
  int32_t tpc = total / 132;
  tpc = tpc < 1 ? 1 : (tpc > tpc_cap ? tpc_cap : tpc);
  // band height of the tile order: as many tile rows as keep the band's A slices (128 K S bytes per tile row) within ~12 MB
  // of the H100's 50 MB L2, at most 16 (K = 1024, S = 7: 13 rows = 11.4 MB; the K = 8192 products of the triangular solves: 1-2 rows)
  int32_t band = (int32_t)((12ll << 20) / (128ll * K * S));
  band = band < 1 ? 1 : (band > 16 ? 16 : band);
  OzParams p{alpha, C, exA + rowA, exB + rowB, ldc, (int32_t)rowA, (int32_t)rowB, (int32_t)(K / OZ_BK), lower,
             tiles_m, tiles_n, total, tpc, tri_rows, beta != 0.0 ? 1 : 0, band};
  // profile: algorithmic (fp64-equivalent) flops of the tiles computed; the int8 work is S (S + 1) / 2 times that
  if (prof_enabled()) prof_begin(stream, (double)total * 2.0 * OZ_BM * OZ_BN * (double)K, 1);
  cudaLaunchAttribute cluster;
  cluster.id = cudaLaunchAttributeClusterDimension;
  cluster.val.clusterDim.x = 2;  // the kernel's CTA pair: one column half of each tile each, A multicast to both
  cluster.val.clusterDim.y = 1;
  cluster.val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * (unsigned)((total + tpc - 1) / tpc));
  cfg.blockDim = dim3(OZ_THREADS);
  cfg.dynamicSmemBytes = OzCfg<S>::SMEM_BYTES;
  cfg.stream = stream;
  cfg.attrs = &cluster;
  cfg.numAttrs = 1;
  const cudaError_t le = cudaLaunchKernelEx(&cfg, oz_gemm_kernel<S>, mA, mB, p);
  if (prof_enabled()) prof_end(stream);
  if (const int rc = cuda_rc(le)) return rc;
  GPK_COUNT_LAUNCH();
  return cuda_rc(cudaGetLastError());
}

}  // namespace

// ---- entry points used by potrf.cu and the C-ABI ----------------------------------------------------------------------
// workspace for `rows` rows of K columns: S int8 planes [S][rows][K] followed by the `rows` row exponents (int32, in 8
// bytes per row)
int64_t oz_ws_bytes(int64_t rows, int64_t K, int32_t S) { return (int64_t)S * rows * K + rows * 8 + 256; }

static inline int32_t* oz_exponents(void* ws, int64_t rows, int64_t K, int32_t S) {
  const uintptr_t p = reinterpret_cast<uintptr_t>(ws) + (uintptr_t)((int64_t)S * rows * K);
  return reinterpret_cast<int32_t*>((p + 255) & ~uintptr_t(255));
}

int oz_slice_panel(const double* P, int64_t ldp, int64_t rows, int64_t K, void* ws, int64_t cap_rows, int32_t S,
                   cudaStream_t stream) {
  if (K % 128 || K > 65536 || rows > cap_rows || ldp % 2 || reinterpret_cast<uintptr_t>(P) % 16) return GPK_ERR_ARG;
  int8_t* planes = static_cast<int8_t*>(ws);
  int32_t* sc = oz_exponents(ws, cap_rows, K, S);
  switch (S) {
    case 5: return oz_launch_slice<5>(P, ldp, rows, K, planes, cap_rows * K, sc, stream);
    case 6: return oz_launch_slice<6>(P, ldp, rows, K, planes, cap_rows * K, sc, stream);
    case 7: return oz_launch_slice<7>(P, ldp, rows, K, planes, cap_rows * K, sc, stream);
    case 8: return oz_launch_slice<8>(P, ldp, rows, K, planes, cap_rows * K, sc, stream);
  }
  return GPK_ERR_ARG;
}

// C[M x N] = beta C + alpha A B^T with A = sliced rows [rowA, rowA + M) of wsA, B = sliced rows [rowB, rowB + N) of wsB
int oz_gemm_sliced(int64_t M, int64_t N, int64_t K, double alpha, const void* wsA, int64_t capA, int64_t rowA,
                   const void* wsB, int64_t capB, int64_t rowB, double beta, double* C, int64_t ldc, int32_t lower,
                   int32_t S, cudaStream_t stream) {
  if (M % OZ_BM || N % OZ_BN || K % 128 || K > 65536 || ldc % 2 || reinterpret_cast<uintptr_t>(C) % 16) return GPK_ERR_ARG;
  if (M == 0 || N == 0) return 0;
  const int8_t* pa = static_cast<const int8_t*>(wsA);
  const int8_t* pb = static_cast<const int8_t*>(wsB);
  const int32_t* sa = oz_exponents(const_cast<void*>(wsA), capA, K, S);
  const int32_t* sb = oz_exponents(const_cast<void*>(wsB), capB, K, S);
#define OZ_CASE(SS)                                                                                                   \
  case SS:                                                                                                            \
    return oz_launch_gemm<SS>(M, N, K, alpha, pa, capA, capA * K, sa, rowA, pb, capB, capB * K, sb, rowB, beta, C, ldc, \
                              lower, stream);
  switch (S) {
    OZ_CASE(5)
    OZ_CASE(6)
    OZ_CASE(7)
    OZ_CASE(8)
  }
#undef OZ_CASE
  return GPK_ERR_ARG;
}

int oz_check_emulation(int32_t S, const void* ws) {
  if (S == 0) return 0;
  return (S < 5 || S > 8 || !ws || reinterpret_cast<uintptr_t>(ws) % 1024) ? GPK_ERR_ARG : 0;
}

static inline int64_t round_up_1k(int64_t x) { return (x + 1023) & ~int64_t(1023); }

// int32 accumulation is exact for K <= 65536 per pass: longer reductions (the sparse path's n = 262144) run as several
// passes over K chunks of this length (a multiple of 128; the last chunk is the remainder), each adding into C
static int64_t oz_k_chunk(int64_t K) {
  const int64_t passes = K > 65536 ? (K + 65535) / 65536 : 1;
  return ((K / passes + 127) / 128) * 128;
}

// scratch of an emulated GEMM with K chunks of kc: A's slices, then (unless B is A) B's from the next 1024-byte boundary
static int64_t oz_gemm_need(int64_t M, int64_t N, int64_t kc, int32_t S, bool same) {
  return same ? oz_ws_bytes(M, kc, S) : round_up_1k(oz_ws_bytes(M, kc, S)) + oz_ws_bytes(N, kc, S);
}

// C = beta C + alpha A B^T on the int8 tensor cores, K chunk by K chunk; `ws` holds oz_gemm_need bytes
static int oz_gemm(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, const double* B, int64_t ldb,
                   double beta, double* C, int64_t ldc, int32_t lower, int32_t S, void* ws, bool same, cudaStream_t stream) {
  const int64_t kc = oz_k_chunk(K);
  void* wsb = static_cast<char*>(ws) + (same ? 0 : round_up_1k(oz_ws_bytes(M, kc, S)));
  int rc;
  for (int64_t k0 = 0; k0 < K; k0 += kc) {
    const int64_t kk = (K - k0 < kc) ? K - k0 : kc;
    if ((rc = oz_slice_panel(A + k0, lda, M, kk, ws, M, S, stream))) return rc;
    if (!same && (rc = oz_slice_panel(B + k0, ldb, N, kk, wsb, N, S, stream))) return rc;
    if ((rc = oz_gemm_sliced(M, N, kk, alpha, ws, M, 0, same ? ws : wsb, same ? M : N, 0, k0 == 0 ? beta : 1.0, C, ldc, lower,
                             S, stream)))
      return rc;
  }
  return 0;
}

int gemm_nt_f64_emulated(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, const double* B,
                         int64_t ldb, double beta, double* C, int64_t ldc, int32_t lower, int32_t S, void* ws, int64_t ws_bytes,
                         cudaStream_t stream) {
  if (!gpk_gemm_nt_oz_ws_bytes(M, N, K, S)) return 0;
  if (M % OZ_BM || N % OZ_BN || K % 128 || lda % 2 || ldb % 2 || ldc % 2) return 0;
  if ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) | reinterpret_cast<uintptr_t>(C)) % 16) return 0;
  const bool same = (A == B && lda == ldb && M >= N);
  if (ws_bytes < oz_gemm_need(M, N, oz_k_chunk(K), S, same)) return 0;
  const int rc = oz_gemm(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, lower, S, ws, same, stream);
  return rc < 0 ? rc : 1;
}

}  // namespace gpk

extern "C" {

int64_t gpk_gemm_nt_oz_ws_bytes(int64_t M, int64_t N, int64_t K, int32_t slices) {
  // worth it only when the product dwarfs the slicing passes and fills the machine
  if (slices < 5 || slices > 8 || M < 256 || N < 256 || K < 256 || (double)M * (double)N * (double)K < 1.5e9) return 0;
  return gpk::oz_gemm_need(M, N, gpk::oz_k_chunk(K), slices, false);
}

int64_t gpk_oz_ws_bytes(int64_t rows, int64_t K, int32_t slices) { return gpk::oz_ws_bytes(rows, K, slices); }

// Host-side evaluation of the emulation GEMM's tile order (the SAME function the kernel runs): tile index t of a launch with
// tiles_m x tiles_n tiles of 128 x 64 -> (tile row, tile column).  Returns the number of tiles of the launch.  Lets the
// CPU test-suite prove that the order is a bijection for every shape without a GPU (an unbounded / wrong order would hang
// or corrupt a launch on the device).
int32_t gpk_debug_oz_tile(int32_t lower, int32_t tiles_m, int32_t tiles_n, int32_t band, int32_t t, int32_t* tm, int32_t* tn) {
  gpk::OzParams p{};
  p.lower = lower;
  p.tiles_m = tiles_m;
  p.tiles_n = tiles_n;
  p.band = band;
  p.tri_rows = lower ? (tiles_m < tiles_n / 2 ? tiles_m : tiles_n / 2) : 0;
  p.total_tiles = lower ? p.tri_rows * (p.tri_rows + 1) + (tiles_m - p.tri_rows) * tiles_n : tiles_m * tiles_n;
  if (t >= 0 && t < p.total_tiles && tm && tn) {
    int a = 0, b = 0;
    gpk::oz_tile(p, t, a, b);
    *tm = a;
    *tn = b;
  }
  return p.total_tiles;
}

int gpk_gemm_nt_f64_oz(int64_t M, int64_t N, int64_t K, double alpha, const double* A, int64_t lda, const double* B,
                       int64_t ldb, double beta, double* C, int64_t ldc, int32_t lower, int32_t slices, void* ws,
                       int64_t ws_bytes, void* stream) {
  const bool same = (A == B && lda == ldb && M >= N);
  if (slices == 0 || gpk::oz_check_emulation(slices, ws) || K <= 0 ||
      ws_bytes < gpk::oz_gemm_need(M, N, gpk::oz_k_chunk(K), slices, same))
    return GPK_ERR_ARG;
  return gpk::oz_gemm(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, lower, slices, ws, same, (cudaStream_t)stream);
}

}  // extern "C"
