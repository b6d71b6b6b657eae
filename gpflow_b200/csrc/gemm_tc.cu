// gemm_tc.cu — fp64 symmetric rank-k update on the Hopper tensor cores (warpgroup MMA, wgmma .s8).
//
//     C[m, n]  -=  A[m, K] * A[0:n, K]^T          (row-major fp64; the Cholesky trailing update)
//
// The integer tensor-core path is far faster than the fp64 one (DMMA), so the fp64 operands are split into balanced
// base-256 digits with a per-row power-of-two scale (an Ozaki-style splitting, planes.cuh):
//
//     a_ik = 2^(e_i - 6) * sum_s 2^(-8 s) d_s(i,k),   d_0 in [-65, 65], d_s in [-128, 127]  (int8),  s = 0..S-1
//
// The digit products accumulate EXACTLY in int32 register accumulators (wgmma m64nNk32 .s32.s8.s8); products with the
// same weight s+t = g < S share one accumulator.  S = 6 adds the (3,3) product in a seventh accumulator (the only
// dropped term whose mean on the diagonal of C is not zero).  A CTA tile is 128 x 32: each of its two consumer
// warpgroups owns 64 rows and NACC = 7 (8 at S = 8) accumulators of 32 columns (112 / 128 registers per thread), and
// issues one m64n32k32 wgmma per digit product: S (S + 1) / 2 (+ 1 at S = 6) per 32-deep k-step.  A comes from
// REGISTERS: per k-step each consumer warp loads its 16 rows of every A plane once (ldmatrix.x4 over the plane's core
// matrices, conflict-free) and feeds them to all S - s products of plane s; only B is read by the tensor core from shared
// memory.  (With both operands in shared memory every A plane was re-read by each of its products: 132 KB of shared-memory
// reads per k-step and SM at S = 6 against 68 KB now, which bounded the kernel at about half of the int8 pipe.)  The A
// fragments are double-buffered across k-steps (single at S = 8), which setmaxnreg makes room for.  The epilogue converts the integer
// accumulators to fp64, recombines them with exact power-of-two weights and the row/column scales, writes the update to a
// shared-memory staging tile and adds it into C with one bulk reduction per 256-byte row (cp.reduce.async.bulk .add.f64,
// performed in L2): the consumers never read C and start the next tile's MMAs while the reductions are in flight.  Error per
// dot product: ~K * (S + 1) * 2^(-8S + 2) relative to the row scales from the dropped products
// (tests/test_digit_slicing_model.py).
//
// Pipeline (per persistent CTA, 384 threads):
//   warps 0-7  two consumer warpgroups (232 registers): A planes -> registers, wgmma with B from shared memory (no-swizzle
//              K-major descriptor), epilogue (each warp stages its 16 rows; lanes 0-15 issue the row reductions); a stage
//              is released by a plain remote mbarrier arrive per CTA of the cluster
//   warp 8     producer (its warpgroup drops to 40 registers; warps 9-11 idle): cp.async.bulk (1-D TMA) of PRE-TILED digit
//              planes global -> shared, mbarrier-tracked stages; in a cluster each CTA fetches 1/CL of every A plane and
//              multicasts it to the CL CTAs sharing the row tile
// The slicing pre-pass (slice_rows_kernel) writes the digit planes directly in the canonical no-swizzle K-major
// shared-memory image (8x16-byte core matrices), so a stage is filled by plain bulk copies.
//
// Replaces the SYRK inside tf.linalg.cholesky (gpflow/models/gpr.py:102 etc.) for the large-K levels
// of the recursion in potrf.cu; small-K levels and ragged shapes use the DMMA kernel of gemm.cu.
#include "tc_common.cuh"
#include "planes.cuh"

namespace gpk {

constexpr int TC_THREADS = 384;                          // 2 consumer warpgroups + 1 producer warpgroup (one working warp)
// registers per thread after setmaxnreg: 8 consumer warps x 232 + 4 producer-group warps x 40 fit the 64 K register file, and
// the 2 + 1 warps of every SM sub-partition its 16 K.  (The launch gets 168: 65536 / 384, rounded down to a multiple of 8.)
constexpr int TC_CONSUMER_REGS = 232, TC_PRODUCER_REGS = 40;
// Epilogue staging: the 128 x 32 fp64 update of a tile, one 256-byte row of C per bulk reduction.  Rows are 320 bytes apart:
// a 16-byte fragment store puts lanes 8 j .. 8 j + 7 on two rows (64 bytes each), which then fill both halves of the 128-byte
// bank window instead of the same half (a 256- or 272-byte pitch keeps them overlapping: two wavefronts per quarter warp).
constexpr int TC_STG_PITCH = 320, TC_STG_BYTES = TC_BM * TC_STG_PITCH;
constexpr int TC_SMEM_BUDGET = 225 * 1024;               // staging + pipeline stages: as many as fit (S planes of A and B per stage)
__host__ __device__ constexpr int tc_stages(int S) {
  const int k = (TC_SMEM_BUDGET - TC_STG_BYTES) / (S * (TC_ATILE + TC_BTILE));
  return k < 6 ? k : 6;
}
constexpr int TC_HEAD_TILES = 128 / TC_BN;               // column tiles of the leading 128-column block

// ------------------------------------------------------------------------------------------------
// scales and slicing
// ------------------------------------------------------------------------------------------------
// static row scales from the ORIGINAL diagonal (planes.cuh): rowscale[i] = 2^(e_i - 6), sqrt(A_ii) < 2^e_i
__global__ void row_exp_kernel(const double* __restrict__ A, int64_t lda, int64_t n, int64_t npad,
                               double* __restrict__ rowscale) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npad) return;
  double sc = 0.0;
  if (i < n) {
    const double d = A[i * lda + i];
    int e = 0;
    if (d > 0.0 && isfinite(d)) e = ilogb(sqrt(d)) + 1;  // e in [-536, 512]: 2^(e - 6) and its inverse are finite
    sc = scalbn(1.0, e - 6);
  }
  rowscale[i] = sc;
}

// dynamic slicing, one CTA per row: rows [row0, row0 + nrows) of the k-range [k0, k0 + K) get the scale of their
// running maximum over that range (the extra rows below the square part; every row when GPK_TC_STATIC=0)
__global__ void __launch_bounds__(256)
slice_rows_kernel(const double* __restrict__ P, int64_t ld, int64_t row0, int64_t nrows, int64_t k0, int64_t K,
                  TcPlanes pl) {
  __shared__ double wmax[8];
  const int64_t i = blockIdx.x;
  tc_slice_row_cta(P + i * ld, row0 + i, k0, K, pl, wmax);
}

struct TcTileIter {  // identical enumeration in every warp role
  // Work unit = CL horizontally adjacent tiles (tm, tnb .. tnb+CL-1), one per CTA of a cluster, so the
  // cluster shares the A tile (multicast).  Order: pass 0 = the "head" units (first 128 columns) of every
  // row tile, pass 1 = the rest: the next diagonal block's inputs are complete early (look-ahead).
  int64_t ntm, ntn;
  int lower, pass, cl, rank;
  int64_t tm, tnb, tn;
  int skip;  // units left to pass over before this cluster's next one: unit i belongs to cluster i % (gridDim.x / cl)
  __device__ TcTileIter(int64_t m, int64_t n, int lower_, int cl_, int rank_)
      : lower(lower_), pass(0), cl(cl_), rank(rank_), tm(0), tnb(-cl_), tn(0), skip((int)blockIdx.x / cl_) {
    ntm = (m + TC_BM - 1) / TC_BM;
    ntn = (n + TC_BN - 1) / TC_BN;
  }
  __device__ int64_t ncols(int64_t t) const {
    const int64_t lim = (t + 1) * (TC_BM / TC_BN);  // column tiles touching the lower triangle of row tile t
    return lower ? (lim < ntn ? lim : ntn) : ntn;
  }
  __device__ bool is_head() const { return pass == 0; }
  // tile index used for LOADING B (clamped: a CTA of a last, partly empty unit loads valid memory and
  // its epilogue writes nothing because its columns are >= n)
  __device__ int64_t tn_load() const { return tn < ntn ? tn : ntn - 1; }
  // false for the padding tiles of a unit that sticks out of the (lower-triangular) tile set: computed, not stored
  __device__ bool valid() const { return tn < ncols(tm); }
  __device__ int64_t head_w() const { return cl > TC_HEAD_TILES ? cl : TC_HEAD_TILES; }
  // advances to this cluster's next unit; false when exhausted.  Every call walks past the units of all other clusters,
  // so the walk counts down instead of taking a 64-bit remainder per unit (that cost microseconds per tile).
  __device__ bool next() {
    for (;;) {
      tnb += cl;
      for (;;) {
        if (pass == 0) {
          const int64_t lim = ncols(tm) < head_w() ? ncols(tm) : head_w();
          if (tm < ntm && tnb >= lim) { ++tm; tnb = 0; continue; }
          if (tm >= ntm) { pass = 1; tm = 0; tnb = head_w(); continue; }
        } else {
          if (tm < ntm && tnb >= ncols(tm)) { ++tm; tnb = head_w(); continue; }
          if (tm >= ntm) return false;
        }
        break;
      }
      if (skip-- == 0) {
        skip = (int)gridDim.x / cl - 1;
        tn = tnb + rank;
        return true;
      }
    }
  }
};

template <int S, int CL>
__global__ void __launch_bounds__(TC_THREADS, 1)
syrk_i8_kernel(TcPlanes pl, int64_t rb0, int64_t kb0, double* __restrict__ C, int64_t ldc, int64_t m, int64_t n, int KB,
               int lower, int* head_flag) {
  // rows of C = global rows 128 rb0 + ..., columns of C = the same rows (C is the block right of the k-range
  // [32 kb0, 32 (kb0 + KB)) on the diagonal); operands come from the digit-plane store (planes.cuh)
  const double* __restrict__ rowscale = pl.rowscale + rb0 * TC_BM;
  int* err = pl.err;
  // even S (6): one more accumulator for the (S/2, S/2) digit product (planes.cuh)
  constexpr bool SQ = (S == 6);
  constexpr int H = S / 2, NACC = S + (SQ ? 1 : 0);
  constexpr bool A2 = S < 8;  // two sets of A fragments (see the consumer's k-step)
  extern __shared__ __align__(1024) uint8_t tc_smem[];
  constexpr uint32_t stage_bytes = (uint32_t)S * (TC_ATILE + TC_BTILE);
  constexpr int TC_STAGES = tc_stages(S);   // S = 6: 6 stages of 30 KB, S = 7: 5 of 35 KB, S = 8: 4 of 40 KB
  uint8_t* stg = tc_smem + TC_STAGES * (size_t)stage_bytes;                  // epilogue staging [128][TC_STG_PITCH]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stg + TC_STG_BYTES);         // full[], empty[]
  const int warp = threadIdx.x >> 5;
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + TC_STAGES);

  if (threadIdx.x == 0) {
    if (blockIdx.x == 0) trace_mark(4, 0);
    for (int i = 0; i < TC_STAGES; ++i) {
      mbar_init(full0 + 8 * i, 1);
      mbar_init(empty0 + 8 * i, 2 * CL);  // both consumer warpgroups of every CTA of the cluster release a stage
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();  // peer barriers initialised before any multicast copy / remote arrive targets them
  // (programmatic dependent launch: everything above overlapped the tail of the preceding kernel; its results -- the digit
  // planes of the panel kernel -- may be read from here on.  A no-op when the launch carried no such dependency.)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (threadIdx.x == 0 && blockIdx.x == 0) trace_mark(4, 10);  // prologue done (barriers, cluster sync)
  const int rank = CL > 1 ? (int)cluster_ctarank() : 0;
  constexpr uint16_t cl_mask = (uint16_t)((1u << CL) - 1);

  if (__all_sync(0xffffffffu, warp >= 8)) {  // vote: the role branch is warp-uniform and the compiler knows it
    // the producer warpgroup hands its registers to the consumers; warps 9-11 have no work
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TC_PRODUCER_REGS));
    // ===== producer (warp 8 runs the loop; one elected lane issues the copies) =====
    if (__all_sync(0xffffffffu, warp == 8)) {
      TcTileIter it(m, n, lower, CL, rank);
      uint32_t st = 0, ph = 0;
      while (it.next()) {
        const int8_t* a_src = pl.tile(rb0 + it.tm, kb0);
        const int64_t tl = it.tn_load();
        const int8_t* b_src = pl.tile(rb0 + tl / (TC_BM / TC_BN), kb0) + (tl % (TC_BM / TC_BN)) * TC_BTILE;
        for (int kb = 0; kb < KB; ++kb) {
          if (CL == 1) mbar_wait(empty0 + 8 * st, ph ^ 1, err, 101);
          else mbar_wait_cluster(empty0 + 8 * st, ph ^ 1, err, 101);
          if (elect_one()) {
            const uint32_t fb = full0 + 8 * st;
            mbar_expect_tx(fb, stage_bytes);
            const uint32_t sa = smem_u32(tc_smem + (size_t)st * stage_bytes);
            const uint32_t sb = sa + S * TC_ATILE;
            if (CL == 1) {
              bulk_g2s(sa, a_src + (size_t)kb * S * TC_ATILE, (uint32_t)S * TC_ATILE, fb);
            } else {
              // each CTA fetches 1/CL of every A plane and multicasts it to the cluster
              constexpr uint32_t part = TC_ATILE / CL;
#pragma unroll
              for (int s2 = 0; s2 < S; ++s2)
                bulk_g2s_mc(sa + s2 * TC_ATILE + rank * part, a_src + ((size_t)kb * S + s2) * TC_ATILE + rank * part, part, fb,
                            cl_mask);
            }
#pragma unroll
            for (int t = 0; t < S; ++t)
              bulk_g2s(sb + t * TC_BTILE, b_src + ((size_t)kb * S + t) * TC_ATILE, TC_BTILE, fb);
          }
          __syncwarp();
          if (++st == TC_STAGES) { st = 0; ph ^= 1; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(TC_CONSUMER_REGS));
    // ===== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====
    const int wg = warp >> 2, wl = warp & 3, lane = threadIdx.x & 31, tid_wg = threadIdx.x & 127;
    TcTileIter it(m, n, lower, CL, rank);
    uint32_t st = 0, ph = 0;
    const bool vec_ok = ((ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
    // a stage is free once this warpgroup's MMAs that read it are complete: one arrive per warpgroup on the stage's empty
    // barrier in every CTA of the cluster (the A planes of every CTA's stage came from all of them)
    auto release = [&](uint32_t s_) {
      if (CL == 1) {
        if (tid_wg == 0) mbar_arrive(empty0 + 8 * s_);
      } else if (tid_wg < CL) {
        mbar_arrive_cluster(empty0 + 8 * s_, (uint32_t)tid_wg);
      }
    };
    // this lane's ldmatrix row address inside a plane: matrix j = lane / 8 is row group 2 wl + (j & 1), k half j / 2
    const uint32_t a_lane = wg * (TC_ATILE / 2) + wl * 512 + ((lane >> 3) & 1) * 256 + (lane >> 4) * 128 + (lane & 7) * 16;
    while (it.next()) {
      uint32_t acc[NACC * 16];
#pragma unroll
      for (int i = 0; i < NACC * 16; ++i) acc[i] = 0u;
      int prev = -1;
      // One k-step.  The warp's 16 rows of every A plane go to registers once (ldmatrix) and feed all of that plane's digit
      // products; B stays in shared memory.  The k-step's MMAs may still read `a` after the commit, so consecutive k-steps
      // alternate between two fragment sets: the set loaded here was last read by the MMAs of two k-steps ago, which
      // wgmma.wait_group 1 of the previous k-step has seen complete.  S = 8 (128 accumulator registers) has room for one
      // set only and waits for the previous k-step's MMAs before it overwrites it.
      auto kstep = [&](uint32_t (&a)[S][4]) {
        mbar_wait(full0 + 8 * st, ph, err, 103);
        if (!A2) wg_wait<0>();
        const uint32_t stage = smem_u32(tc_smem + (size_t)st * stage_bytes);
#pragma unroll
        for (int s = 0; s < S; ++s) ldsm_x4(a[s], stage + s * TC_ATILE + a_lane);
        const uint64_t bd = wg_desc(stage + S * TC_ATILE, 128, 256);
        wg_fence();
#pragma unroll
        for (int s = 0; s < S; ++s) {
          // digit products (s, t) with s + t < S into accumulator s + t; at S = 6 also (H, H): the square term, accumulator S
          const int c = (SQ && s == H) ? H + 1 : S - s;
#pragma unroll
          for (int t = 0; t < c; ++t)
            WgmmaS8<TC_BN>::mma_rs(acc + 16 * (s + t), a[s], bd + (uint64_t)(t * (TC_BTILE >> 4)), 1u);
        }
        wg_commit();
        wg_wait<1>();  // the previous k-step's MMAs are complete: its stage may be refilled
        if (prev >= 0) release((uint32_t)prev);
        prev = (int)st;
        if (++st == TC_STAGES) { st = 0; ph ^= 1; }
      };
      uint32_t af[A2 ? 2 : 1][S][4];
      if (A2) {
        int kb = 0;
        for (; kb + 1 < KB; kb += 2) {
          kstep(af[0]);
          kstep(af[1 % (A2 ? 2 : 1)]);
        }
        if (kb < KB) kstep(af[0]);
      } else {
        for (int kb = 0; kb < KB; ++kb) kstep(af[0]);  // (unrolled by two, ptxas serialises the S = 8 wgmmas)
      }
      // Full 32-column tiles of a 16-byte aligned C take the bulk-reduction epilogue (below).  Its column scales are loaded
      // while the last k-step's MMAs run, so that their L2 latency passes behind them.  (Loaded before the main loop, or
      // with the row scales as well, they keep registers live that S = 7 then spills.)
      const int64_t colb = it.tn * TC_BN;
      const bool bulk = vec_ok && colb + TC_BN <= n;
      double2 csv[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        csv[q] = bulk ? __ldg(reinterpret_cast<const double2*>(rowscale + colb + 8 * q + 2 * (lane & 3))) : make_double2(0.0, 0.0);
      wg_wait<0>();
      wg_keep(acc, NACC * 16);
      if (prev >= 0) release((uint32_t)prev);
      const bool tr0 = blockIdx.x == 0 && threadIdx.x == 0 && it.is_head() && it.tm == 0;  // (first tile of CTA 0)
      if (tr0) trace_mark(4, 13);  // accumulators complete

      // ---- epilogue: fragment element j = 4 q + 2 h + e is row 16 wl + lane / 4 + 8 h, column 8 q + 2 (lane % 4) + e ----
      // Bulk form: the update goes to the warp's 16 staging rows and lanes 0-15 add one row each into C with a bulk
      // reduction (performed in L2); the warp never reads C and goes straight on to the next tile.  Every element of C
      // receives exactly one update per launch and u = (-rs_i rs_j) v is an exact power-of-two scaling of v, so round(C + u)
      // is what the read-modify-write below (still used at a ragged right edge or for an unaligned C) stores.
      if (bulk) {
        bulk_wait_read<0>();  // the previous tile's reductions have read the staging rows
        __syncwarp();
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = 16 * warp + (lane >> 2) + 8 * h;  // row in the tile (warp = 4 wg + wl)
        const int64_t row = it.tm * TC_BM + r;
        if (!(row < m && it.valid())) continue;
        const double rs = -__ldg(rowscale + row);
        double* crow = C + row * ldc;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int64_t col = colb + 8 * q + 2 * (lane & 3);
          double v[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            double a = 0.0, w = 1.0;
#pragma unroll
            for (int g = 0; g < NACC; ++g) {
              a = fma(tc_int_to_double((int)acc[g * 16 + 4 * q + 2 * h + e]), w, a);
              w *= 0.00390625;  // 2^-8 (radix 256)
            }
            v[e] = a;
          }
          if (bulk) {
            const double2 s2 = csv[q];
            *reinterpret_cast<double2*>(stg + r * TC_STG_PITCH + (8 * q + 2 * (lane & 3)) * 8) =
                make_double2((rs * s2.x) * v[0], (rs * s2.y) * v[1]);
          } else if (vec_ok && col + 1 < n) {
            const double2 s2 = __ldg(reinterpret_cast<const double2*>(rowscale + col));
            double2 o = *reinterpret_cast<double2*>(crow + col);
            o.x += (rs * s2.x) * v[0];
            o.y += (rs * s2.y) * v[1];
            *reinterpret_cast<double2*>(crow + col) = o;
          } else {  // ragged right edge / unaligned C
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (col + e < n) crow[col + e] += (rs * __ldg(rowscale + col + e)) * v[e];
          }
        }
      }
      if (bulk) {
        fence_proxy_async_shared();  // this thread's staging stores before the bulk reductions that read them
        __syncwarp();
        if (lane < 16) {
          const int r = 16 * warp + lane;
          const int64_t row = it.tm * TC_BM + r;
          if (row < m && it.valid()) bulk_reduce_add_f64(C + row * ldc + colb, smem_u32(stg + r * TC_STG_PITCH), TC_BN * 8);
          bulk_commit();
        }
      }
      if (tr0) trace_mark(4, 15);  // update stored (read-modify-write) or its reductions issued
      if (head_flag && it.is_head()) {
        // flag[1] is what the look-ahead leaf acquires before it reads the next diagonal block of C: a tile that overlaps
        // that block is published once both consumer warpgroups' updates are complete in global memory.  flag[0] only
        // counts the head tiles (nothing waits on it), so the other head tiles go on without waiting for their reductions.
        const int u = diag_units_tile(it.tm * TC_BM, it.tn * TC_BN, TC_BM, TC_BN, m, n);
        if (u) {
          if (bulk) {  // the reductions must be complete, not just issued
            bulk_wait<0>();
            fence_proxy_async_global();
          }
          __threadfence();
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (tr0) trace_mark(4, 16);  // update complete in global memory (the tile may be published)
          if (threadIdx.x == 0) {
            trace_mark(4, 1);  // a head tile published
            atomicAdd(head_flag, 1);
            atomicAdd(head_flag + 1, u);  // progress on the next diagonal block
          }
        } else if (threadIdx.x == 0) {
          atomicAdd(head_flag, 1);
        }
      }
    }
    bulk_wait<0>();  // the staging rows stay valid, and the CTA resident, until every reduction is complete
  }

  __syncthreads();
  if (threadIdx.x == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1)) trace_mark(4, blockIdx.x == 0 ? 2 : 3);
  if (CL > 1) cluster_sync_all();  // no CTA leaves while a peer may still multicast into its shared memory / arrive on it
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
// GPK_TC_SLICES pins the number of digit planes (6..8); 0 = chosen per factorisation (potrf.cu::pick_slices)
int tc_slices() {
  static int s = -1;
  if (s < 0) {
    const char* e = getenv("GPK_TC_SLICES");
    s = e ? atoi(e) : 0;
    if (s != 0 && s < 6) s = 6;
    if (s > TC_MAXS) s = TC_MAXS;
  }
  return s;
}

int trace_set_tc(TraceBuf tb) {
  GPK_CUDA_OK(cudaMemcpyToSymbol(g_trace, &tb, sizeof(tb)));
  return 0;
}

bool tc_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("GPK_FP64_ENGINE");
    v = (e && (strcmp(e, "dmma") == 0 || strcmp(e, "simt") == 0)) ? 0 : 1;
  }
  return v == 1;
}

static bool tc_static_scales() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("GPK_TC_STATIC"); v = (e && e[0] == '0') ? 0 : 1; }
  return v == 1;
}

static bool tc_rect() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("GPK_TC_RECT"); v = (e && e[0] == '1') ? 1 : 0; }
  return v == 1;
}

static size_t tc_tiles_total(int64_t rbt, int64_t nbk) {
  return (size_t)(tc_rect() ? rbt * 4 * nbk : plane_prefix(rbt, nbk));
}

size_t tc_planes_bytes(int64_t n, int64_t rows) {
  const int64_t nbk = (n + TC_BM - 1) / TC_BM, rbt = (rows + TC_BM - 1) / TC_BM;
  return align_up(tc_tiles_total(rbt, nbk) * TC_MAXS * TC_ATILE, 256) + align_up((size_t)rbt * TC_BM * sizeof(double), 256) + 256;
}

TcPlanes tc_planes_layout(void* ws, int64_t n, int64_t rows, int S) {
  const int64_t nbk = (n + TC_BM - 1) / TC_BM, rbt = (rows + TC_BM - 1) / TC_BM;
  TcPlanes pl;
  pl.planes = (int8_t*)ws;
  pl.rowscale = (double*)((char*)ws + align_up(tc_tiles_total(rbt, nbk) * TC_MAXS * TC_ATILE, 256));
  pl.rect = tc_rect();
  pl.err = (int*)((char*)pl.rowscale + align_up((size_t)rbt * TC_BM * sizeof(double), 256));
  pl.S = S;
  pl.nbk = nbk;
  pl.n_sq = n;
  pl.is_static = tc_static_scales();
  return pl;
}

int tc_row_exponents(const double* A, int64_t lda, const TcPlanes& pl, cudaStream_t st) {
  const int64_t npad = (pl.n_sq + TC_BM - 1) / TC_BM * TC_BM;
  ProfScope ps(PROF_MISC, st);
  row_exp_kernel<<<(unsigned)((npad + 255) / 256), 256, 0, st>>>(A, lda, pl.n_sq, npad, pl.rowscale);
  GPK_LAUNCH_OK();
  return 0;
}

int tc_slice_rows(const double* P, int64_t ld, int64_t row0, int64_t nrows, int64_t k0, int64_t K, const TcPlanes& pl,
                  cudaStream_t st) {
  if (nrows <= 0) return 0;
  GPK_CHECK_ARG(K % TC_KB == 0 && k0 % TC_KB == 0, "tc_slice_rows: k-range must be a multiple of 32");
  ProfScope ps(PROF_MISC, st);
  slice_rows_kernel<<<(unsigned)nrows, 256, 0, st>>>(P, ld, row0, nrows, k0, K, pl);
  GPK_LAUNCH_OK();
  return 0;
}

static int tc_num_sms() {  // of the CURRENT device (a process may drive several)
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 132;
}

// C[m,n] -= L[r0:r0+m, k0:k0+K] L[r0:r0+n, k0:k0+K]^T (lower tiles only if `lower`); K, k0 % 32 == 0, r0 % 128 == 0, n <= m.
int syrk_tc_planes(double* C, int64_t ldc, int64_t m, int64_t n, const TcPlanes& pl, int64_t r0, int64_t k0, int64_t K,
                   int lower, cudaStream_t st, const GemmOpts* opts) {
  const int S = pl.S;
  int* hf = opts ? opts->head_flag : nullptr;
  GPK_CHECK_ARG(K % TC_KB == 0 && K > 0 && n <= m && r0 % TC_BM == 0 && k0 % TC_KB == 0,
                "syrk_tc: unsupported shape m=%lld n=%lld K=%lld r0=%lld k0=%lld", (long long)m, (long long)n, (long long)K,
                (long long)r0, (long long)k0);
  const int64_t rb0 = r0 / TC_BM, kb0 = k0 / TC_KB;
  const size_t smem = tc_stages(S) * (size_t)S * (TC_ATILE + TC_BTILE) + TC_STG_BYTES + 256;
  // Clusters of 2 CTAs multicast the shared A tile (it is 4x the B tile); GPK_TC_CLUSTER=1 disables, =4 widens.
  static const int cl_env = []() {
    const char* e = getenv("GPK_TC_CLUSTER");
    return (e && e[0] == '1') ? 1 : (e && e[0] == '4') ? 4 : 2;
  }();
  const int cl = (opts && opts->tc_cluster) ? opts->tc_cluster : cl_env;
  GPK_CHECK_ARG(cl == 1 || cl == 2 || cl == 4, "syrk_tc: cluster width %d is not 1, 2 or 4", cl);
  // number of work units (CL adjacent tiles)
  const int64_t ntm = (m + TC_BM - 1) / TC_BM, ntn = (n + TC_BN - 1) / TC_BN;
  int64_t nunits = 0;
  for (int64_t t = 0; t < ntm; ++t) {
    const int64_t lim = (t + 1) * (TC_BM / TC_BN);
    const int64_t nc = lower ? (lim < ntn ? lim : ntn) : ntn;
    nunits += (nc + cl - 1) / cl;
  }
  int grid = tc_num_sms() - (hf ? 1 : 0);  // look-ahead: leave one SM for the concurrent leaf kernel
  grid = grid / cl * cl;
  if (nunits * cl < grid) grid = (int)(nunits * cl);
  if (grid < 1) return 0;
  const int KBn = (int)(K / TC_KB);
  // issued int8 MACs: every tile of every unit (padding tiles included) x k-steps x S(S+1)/2 digit products
  ProfScope ps(PROF_TC, st, (double)nunits * cl * KBn * (S * (S + 1) / 2 + (S == 6 ? 1 : 0)) * (double)(TC_BM * TC_BN * TC_KB));
  static const bool pdl = []() { const char* e = getenv("GPK_TC_PDL"); return e && e[0] == '1'; }();  // off: see potrf_panel_kernel
  auto launch = [&](auto kern) -> int {
    GPK_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)cl;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl ? 2 : 1;
    GPK_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, pl, rb0, kb0, C, ldc, m, n, KBn, lower, hf));
    count_launch();
    return 0;
  };
#define GPK_TC_PICK(CC) (S == 6 ? launch(syrk_i8_kernel<6, CC>) : S == 7 ? launch(syrk_i8_kernel<7, CC>) : launch(syrk_i8_kernel<8, CC>))
  if (cl == 4) return GPK_TC_PICK(4);
  if (cl == 2) return GPK_TC_PICK(2);
  return GPK_TC_PICK(1);
#undef GPK_TC_PICK
}

// gpk_debug_syrk_i8: one update as potrf issues it for rows with dynamic (row-maximum) scales.  The plane store has the
// layout of a factorisation with n_sq = r0, so every operand row is an extra row holding all r0 / 32 k-blocks; only the row
// blocks of the m operand rows are allocated (the tile and row-scale bases are offset by the r0 rows above them, which the
// kernels never touch).  A points at the first operand row.
int tc_debug_syrk(const double* A, int64_t lda, int64_t r0, int64_t k0, int64_t K, double* C, int64_t ldc, int64_t m,
                  int64_t n, int lower, int S, int cluster, double* rowscale_out, int* head_flag, cudaStream_t st) {
  GPK_CHECK_ARG(A && C && m > 0 && n > 0 && n <= m && K > 0 && k0 >= 0 && r0 % TC_BM == 0 && k0 % TC_KB == 0 &&
                    K % TC_KB == 0 && k0 + K <= r0 && lda >= k0 + K && ldc >= n && S >= 6 && S <= TC_MAXS &&
                    (cluster == 1 || cluster == 2 || cluster == 4) && K * S * 16384 < (1ll << 31),
                "debug_syrk_i8: unsupported arguments (m=%lld n=%lld r0=%lld k0=%lld K=%lld S=%d cluster=%d)", (long long)m,
                (long long)n, (long long)r0, (long long)k0, (long long)K, S, cluster);
  const int64_t nbk = r0 / TC_BM, rb_end = nbk + (m + TC_BM - 1) / TC_BM;
  const size_t tile_bytes = (size_t)S * TC_ATILE;
  const size_t skip = tc_tiles_total(nbk, nbk) * tile_bytes;                       // tiles of the rows above r0
  const size_t plane_bytes = align_up(tc_tiles_total(rb_end, nbk) * tile_bytes - skip, 256);
  const size_t rs_bytes = align_up((size_t)(rb_end - nbk) * TC_BM * sizeof(double), 256);
  void* ws = nullptr;
  GPK_CUDA_OK(cudaMalloc(&ws, plane_bytes + rs_bytes + 256));
  TcPlanes pl;
  pl.planes = reinterpret_cast<int8_t*>(reinterpret_cast<uintptr_t>(ws) - skip);
  pl.rowscale = reinterpret_cast<double*>(reinterpret_cast<uintptr_t>(ws) + plane_bytes - (size_t)r0 * sizeof(double));
  pl.err = reinterpret_cast<int*>(reinterpret_cast<char*>(ws) + plane_bytes + rs_bytes);
  pl.S = S;
  pl.nbk = nbk;
  pl.n_sq = r0;
  pl.is_static = tc_static_scales();
  pl.rect = tc_rect();
  GemmOpts opts;
  opts.head_flag = head_flag;
  opts.tc_cluster = cluster;
  auto run = [&]() -> int {
    GPK_CUDA_OK(cudaMemsetAsync(pl.err, 0, sizeof(int), st));
    GPK_TRY(tc_slice_rows(A + k0, lda, r0, m, k0, K, pl, st));
    GPK_TRY(syrk_tc_planes(C, ldc, m, n, pl, r0, k0, K, lower, st, &opts));
    if (rowscale_out)
      GPK_CUDA_OK(cudaMemcpyAsync(rowscale_out, pl.rowscale + r0, (size_t)m * sizeof(double), cudaMemcpyDeviceToDevice, st));
    GPK_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
  };
  const int rc = run();
  cudaStreamSynchronize(st);
  cudaFree(ws);
  return rc;
}

}  // namespace gpk
