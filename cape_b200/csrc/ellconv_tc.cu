// Tensor-core (wgmma, sm_90a) version of the fused ELL-gather Chebyshev convolution, and of the same contraction for
// calls whose terms are all plain tensors (identity operators: 1x1 convs, the split convolution forms, the GroupNorm
// blocks' linear layers).
//
// Same math and epilogues as ellconv.cu, but the [128 x Fin*K] x [Fin*K x BN] contraction runs on the tensor cores
// with fp32 accuracy by 3xTF32 error compensation:  a = a_hi + a_lo (a_hi = top 19 bits, a_lo = the exact remainder),
// acc += a_hi*b_hi + a_lo*b_hi + a_hi*b_lo with fp32 accumulation; the dropped a_lo*b_lo term is ~2^-22 relative.
//
// The kernel is persistent: one CTA per SM (at most one fits) loops over 128-row x BN-column output tiles, and runs
// four warpgroups around a ring of shared-memory stages:
//  - warpgroups 0 and 1, the producers, gather the Chebyshev-basis chunk A[128 rows x 32 k] from neighbour rows
//    (float4 loads, same ELL tables and row mapping as the SIMT path) or load it from a plain operand, split it into
//    hi/lo and store it in the swizzled K-major layout of the next free stage.  The weight chunk B[BN x 32 k] (K-major
//    copy of W) comes by TMA, issued by one producer before the gather, straight into the stage's hi tile in the same
//    layout; after the gather the producers split it in place into hi/lo.  Then they arrive on the stage's `full`
//    mbarrier;
//  - warpgroups 2 and 3, the consumers, each own 64 output rows: wait on `full`, issue wgmma m64nBNk8 for the chunk,
//    wait for it, add the chunk's sum into the running accumulator and release the stage on its `empty` mbarrier; at
//    the tile's last chunk they run the epilogue from the accumulator registers.
// The producers run up to STAGES chunks ahead, across tile boundaries: the ring's stage and phase run on over the
// CTA's tiles, so the gather of the next tile overlaps the MMAs and the epilogue of the previous one (most launches
// of the step have only 2-8 chunks per tile, which a one-tile CTA spends in ramp and drain).  The two consumers never
// wait for each other.  setmaxnreg moves registers from the producers to the consumers, which hold the accumulators.
// Two producer warpgroups, not one, and each producer thread gathers both of its row pairs at once (16 neighbour-row
// loads in flight): the gather is latency-bound on L2.  The weights take no producer registers while it runs.
// Tiles are handed out by ticket (an atomic counter of the topology handle) in the order row tile, then column tile
// fastest, so the CTAs of one row tile run together and read its source rows from L2 rather than from HBM once per
// column tile, and a CTA that starts late (the weight-gradient stream holding its SM) simply takes fewer tiles.
//
// Every chunk's products go to a fresh register accumulator that is added to the running sum in fp32 with
// round-to-nearest, so the tensor core's truncating accumulation chain is one chunk (12 MMAs) long instead of the whole
// reduction: long reductions would otherwise drift from the fp64 truth by more than 1e-4 (cape_conv_args.precise
// has no effect).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <algorithm>
#include <cstring>
#include <type_traits>
#include "common.cuh"
#include "ellconv_params.cuh"
#include "tc_common.cuh"

namespace cape {

namespace {

using namespace tc;

constexpr int CONV_THREADS = 512;             // two producer warpgroups + two consumer warpgroups
constexpr int PRODUCER_THREADS = 256;
constexpr int CONSUMER_THREADS = 256;
// per-thread registers after setmaxnreg: 256 * PRODUCER_REGS + 256 * CONSUMER_REGS <= 512 * 128 (the launch budget
// of a 512-thread CTA)
constexpr int PRODUCER_REGS = 112;
constexpr int CONSUMER_REGS = 144;
constexpr int GATHER_PAIRS = 2;               // row pairs each producer thread gathers at once
constexpr int A_TILE = BM * 128;              // 128 rows x 32 fp32
constexpr int QS_MAX_FLOATS = 8192;           // condition vectors of the tile's samples and columns
constexpr int BAR_BYTES = 256;                // the ring's mbarriers and tile slots
constexpr int SMEM_MAX = 227 * 1024;          // dynamic shared memory per CTA on sm_90

template <int BN, bool DUAL>
struct ConvCfg {
  static constexpr int B_TILE = BN * 128;
  static constexpr int STAGE = 2 * A_TILE + (DUAL ? 4 : 2) * B_TILE;
  // as many stages (up to 4) as fit beside the largest condition-vector buffer
  static constexpr int FIT = (SMEM_MAX - 1024 - BAR_BYTES - QS_MAX_FLOATS * 4) / STAGE;
  static constexpr int STAGES = FIT < 4 ? FIT : 4;
  static constexpr int RING = STAGES * STAGE;
  static_assert(STAGES >= 3, "the ring needs at least three stages");
  static_assert(3 * STAGES * 8 + STAGES * 4 <= BAR_BYTES, "mbarrier area too small");
};

// TMA descriptors of the terms' K-major weight copies, encoded at launch: w[t][0] maps wT and w[t][1] w2T of term t,
// each as a [ncols x F] tensor (row stride wT_stride) read in boxes of 32 k x BN columns with the 128-byte swizzle,
// the layout of the stage's weight tiles; the zero fill beyond F and ncols pads the last chunk and column tile
struct WeightMaps {
  CUtensorMap w[CAPE_MAX_TERMS][2];
};

// Gathers rows (ra[i], rb[i]) for NP pairs: the producers' copy of ell_gather4_pair (NP = 1), which this one matches
// tap for tap; written for NP pairs at once so that more loads can be put in flight when registers allow.  Each
// pair stops when both of its rows are exhausted, and an exhausted row of a live pair adds 0 * (row 0), exactly as
// ell_gather4_pair does for one pair.
template <int NP>
__device__ __forceinline__ void ell_gather4_pairs(const OpView& op, const int (&ra)[NP], const int (&rb)[NP],
                                                  const float* (&base_a)[NP], const float* (&base_b)[NP],
                                                  size_t stride, float4 (&va)[NP], float4 (&vb)[NP]) {
  const int nb = op.width >> 2;
  int4 ia[NP], ib[NP];
#pragma unroll
  for (int q = 0; q < NP; ++q) {
    ia[q] = __ldg(reinterpret_cast<const int4*>(op.idx + (size_t)ra[q] * op.width));
    ib[q] = __ldg(reinterpret_cast<const int4*>(op.idx + (size_t)rb[q] * op.width));
  }
  for (int b = 0; b < nb; ++b) {
    bool any = false;
#pragma unroll
    for (int q = 0; q < NP; ++q) any |= ia[q].x >= 0 || ib[q].x >= 0;
    if (!any) break;
#pragma unroll
    for (int q = 0; q < NP; ++q) {
      const bool da = ia[q].x >= 0, db = ib[q].x >= 0;
      if (!da && !db) continue;
      float4 wa = make_float4(0.f, 0.f, 0.f, 0.f), wb = make_float4(0.f, 0.f, 0.f, 0.f);
      if (da) wa = __ldg(reinterpret_cast<const float4*>(op.w + (size_t)ra[q] * op.width) + b);
      if (db) wb = __ldg(reinterpret_cast<const float4*>(op.w + (size_t)rb[q] * op.width) + b);
      int4 na = make_int4(-1, -1, -1, -1), nbx = make_int4(-1, -1, -1, -1);
      if (b + 1 < nb) {
        na = __ldg(reinterpret_cast<const int4*>(op.idx + (size_t)ra[q] * op.width) + b + 1);
        nbx = __ldg(reinterpret_cast<const int4*>(op.idx + (size_t)rb[q] * op.width) + b + 1);
      }
      const float* pa = base_a[q];
      const float* pb = base_b[q];
      const float4 a0 = ldg4(pa + (size_t)max(ia[q].x, 0) * stride), a1 = ldg4(pa + (size_t)max(ia[q].y, 0) * stride);
      const float4 a2 = ldg4(pa + (size_t)max(ia[q].z, 0) * stride), a3 = ldg4(pa + (size_t)max(ia[q].w, 0) * stride);
      const float4 b0 = ldg4(pb + (size_t)max(ib[q].x, 0) * stride), b1 = ldg4(pb + (size_t)max(ib[q].y, 0) * stride);
      const float4 b2 = ldg4(pb + (size_t)max(ib[q].z, 0) * stride), b3 = ldg4(pb + (size_t)max(ib[q].w, 0) * stride);
      fma4(va[q], wa.x, a0); fma4(va[q], wa.y, a1); fma4(va[q], wa.z, a2); fma4(va[q], wa.w, a3);
      fma4(vb[q], wb.x, b0); fma4(vb[q], wb.y, b1); fma4(vb[q], wb.z, b2); fma4(vb[q], wb.w, b3);
      ia[q] = na; ib[q] = nbx;
    }
  }
}

// PASS: the call has pass-through terms (added in the epilogue); a separate instantiation, so that the kernels of the
// other calls compile exactly as without them.
// Tiles come from *counter, which is 0 at the start of a launch: each CTA draws tickets until one is past the last
// tile, so a launch draws exactly ntiles + gridDim.x tickets, and the CTA that draws the last one resets the counter
// for the next launch of the handle.
template <int BN, bool DUAL, bool PASS>
__global__ void __launch_bounds__(CONV_THREADS, 1) conv_wg_kernel(const __grid_constant__ ConvParams p,
                                                                  const __grid_constant__ WeightMaps maps, int nqs,
                                                                  int ncol_tiles, int ntiles, unsigned* counter) {
  using Cfg = ConvCfg<BN, DUAL>;
  constexpr int S = Cfg::STAGES;
  constexpr int NA = BN / 2;                  // accumulator registers per consumer thread
  extern __shared__ uint8_t smem_raw[];
  char* smem = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::RING);
  uint64_t* empty = full + S;
  uint64_t* wfull = empty + S;                // the stage's weight tiles have landed (TMA transaction bytes)
  // tile_slot[s]: the tile whose first chunk stage s holds (-1: no more tiles), set before the stage's `full` arrive;
  // one per stage, as the producers run up to a tile ahead of the consumers
  int* tile_slot = reinterpret_cast<int*>(wfull + S);
  float* qs = reinterpret_cast<float*>(smem + Cfg::RING + BAR_BYTES);

  const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127;

  // the reduction: 32-deep chunks over all terms (a term of F = 0 still takes one all-zero chunk)
  int nchunks = 0;
  for (int t = 0; t < p.nterms; ++t) nchunks += max(1, (p.terms[t].F + BK - 1) / BK);

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], PRODUCER_THREADS);  // every producer thread
      mbar_init(&empty[s], 8);                // one lane per consumer warp
      mbar_init(&wfull[s], 1);                // the producer that issues the stage's weight loads
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (tid < PRODUCER_THREADS) {
    // =========================== producers ===========================
    setmaxnreg_dec<PRODUCER_REGS>();
    // 8 threads per 128-byte tile row (one float4 of k each), 32 row slots; rows rs + 32 i, gathered in the pairs
    // (rs, rs + 32) and (rs + 64, rs + 96): the row mapping of the SIMT kernels, so each row's taps add in their order
    const int l8 = tid & 7, rs = tid >> 3;
    constexpr int ROWS[4] = {0, 32, 64, 96};
    uint32_t it = 0;                          // the CTA's running chunk count: ring stage it % S, phase (it / S) & 1
    unsigned next = 0;
    if (tid == 0) next = atomicAdd(counter, 1u);
    for (;;) {
      // the stage of the tile's first chunk takes the tile's index, for the other producers and the consumers
      mbar_wait(&empty[it % S], ((it / S) & 1) ^ 1);
      if (tid == 0) tile_slot[it % S] = next < (unsigned)ntiles ? (int)next : -1;
      named_bar_sync(2, PRODUCER_THREADS);
      const int tile = tile_slot[it % S];     // not rewritten before the consumers have released this stage
      if (tile < 0) {                         // no more tiles
        if (tid == 0 && next == (unsigned)ntiles + gridDim.x - 1) *counter = 0u;   // the launch's last ticket
        mbar_arrive(&full[it % S]);
        return;
      }
      if (tid == 0) next = atomicAdd(counter, 1u);   // the following tile's ticket, in flight during this tile
      const int ct = tile % ncol_tiles;
      const long long row0 = (long long)(tile / ncol_tiles) * BM;
      const int col0 = ct * BN;
      int rn[4], rr[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const long long R = row0 + rs + ROWS[i];
        if (R < p.total_rows) { rn[i] = (int)(R / p.rows_out); rr[i] = (int)(R % p.rows_out); }
        else { rn[i] = -1; rr[i] = 0; }
      }
      const bool do_stash = ct == 0;          // one column tile writes the basis copies
      int t = 0, f0 = 0;
      for (int j = 0; j < nchunks; ++j, ++it) {
        const int stage = it % S;
        mbar_wait(&empty[stage], ((it / S) & 1) ^ 1);
        char* a_hi = smem + (size_t)stage * Cfg::STAGE;
        char* a_lo = a_hi + A_TILE;
        char* b_hi = a_lo + A_TILE;
        char* b_lo = b_hi + Cfg::B_TILE;
        const TermDev& tm = p.terms[t];
        const int f = f0 + l8 * 4;
        // the weight chunk first, by TMA into the hi tiles: it lands while the gather runs
        const bool has2 = DUAL && tm.w2T != nullptr;
        if (tid == 0) {
          mbar_arrive_expect_tx(&wfull[stage], (has2 ? 2 : 1) * Cfg::B_TILE);
          tma_load_2d(b_hi, &maps.w[t][0], f0, col0, &wfull[stage]);
          if (has2) tma_load_2d(b_lo + Cfg::B_TILE, &maps.w[t][1], f0, col0, &wfull[stage]);
        }
#pragma unroll
        for (int h = 0; h < 2 / GATHER_PAIRS; ++h) {  // GATHER_PAIRS pairs (ROWS[2q], ROWS[2q + 1]) at a time
          constexpr int NP = GATHER_PAIRS;
          float4 va[NP], vb[NP];
#pragma unroll
          for (int q = 0; q < NP; ++q) { va[q] = make_float4(0.f, 0.f, 0.f, 0.f); vb[q] = va[q]; }
          if (f < tm.F) {
            // invalid (beyond-the-end) rows gather sample 0 / row 0 and are zeroed afterwards
            const float* base_a[NP];
            const float* base_b[NP];
            int ra[NP], rb_[NP];
#pragma unroll
            for (int q = 0; q < NP; ++q) {
              const int ia = 2 * (h * NP + q);
              base_a[q] = tm.src + (size_t)max(rn[ia], 0) * tm.src_rows * tm.src_stride + f;
              base_b[q] = tm.src + (size_t)max(rn[ia + 1], 0) * tm.src_rows * tm.src_stride + f;
              ra[q] = rr[ia]; rb_[q] = rr[ia + 1];
            }
            if (tm.op.idx == nullptr) {
#pragma unroll
              for (int q = 0; q < NP; ++q) {
                va[q] = ldg4(base_a[q] + (size_t)ra[q] * tm.src_stride);
                vb[q] = ldg4(base_b[q] + (size_t)rb_[q] * tm.src_stride);
              }
            } else {
              ell_gather4_pairs<NP>(tm.op, ra, rb_, base_a, base_b, (size_t)tm.src_stride, va, vb);
            }
          }
#pragma unroll
          for (int q = 0; q < NP; ++q) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int i = 2 * (h * NP + q) + e;
              float4 v = e == 0 ? va[q] : vb[q];
              if (rn[i] < 0) v = make_float4(0.f, 0.f, 0.f, 0.f);
              const int row = rs + ROWS[i];
              if (f < tm.F && tm.stash != nullptr && do_stash && rn[i] >= 0)   // basis rows for the weight gradient
                *reinterpret_cast<float4*>(tm.stash + (size_t)(row0 + row) * tm.stash_stride + f) = v;
              split_store4(v, a_hi, a_lo, (uint32_t)(row * 128 + ((l8 ^ (row & 7)) << 4)));
            }
          }
        }
        // the weight chunk, split in place: hi = tf32_hi(w), lo = w - hi (zeros for a term without w2T)
        mbar_wait(&wfull[stage], (it / S) & 1);
#pragma unroll
        for (int i = 0; i < BN / 32; ++i) {
          const int cl = rs + 32 * i;
          const uint32_t off = (uint32_t)(cl * 128 + ((l8 ^ (cl & 7)) << 4));
          split_store4(*reinterpret_cast<const float4*>(b_hi + off), b_hi, b_lo, off);
          if (DUAL) {
            char* b2_hi = b_lo + Cfg::B_TILE;
            const float4 v2 = has2 ? *reinterpret_cast<const float4*>(b2_hi + off) : make_float4(0.f, 0.f, 0.f, 0.f);
            split_store4(v2, b2_hi, b2_hi + Cfg::B_TILE, off);
          }
        }
        fence_proxy_async();                  // generic-proxy smem writes -> visible to the tensor core's (async) proxy
        mbar_arrive(&full[stage]);
        f0 += BK;
        if (f0 >= tm.F) { f0 = 0; ++t; }
      }
    }
  }

  // =========================== consumers ===========================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int cw = wg - 2, ctid = tid - PRODUCER_THREADS;
  const bool linear = p.epilogue == CAPE_EPI_LINEAR;
  const bool use_aux = p.epilogue == CAPE_EPI_SLOPE || p.epilogue == CAPE_EPI_DUALMASK;
  uint32_t it = 0;                            // as the producers' count
  for (;;) {
    mbar_wait(&full[it % S], (it / S) & 1);   // the tile's first chunk carries its index
    const int tile = tile_slot[it % S];
    if (tile < 0) return;

    // one chunk accumulator for both running sums where two would not fit beside them (DUAL, BN = 64): the second
    // sum's MMAs then wait for the first one's add
    constexpr bool ONE_PART = DUAL && BN == 64;
    float acc0[NA], acc1[DUAL ? NA : 1], part0[NA], part1[DUAL && !ONE_PART ? NA : 1];
#pragma unroll
    for (int i = 0; i < NA; ++i) { acc0[i] = 0.f; if (DUAL) acc1[i] = 0.f; }

    for (const uint32_t end = it + nchunks; it != end; ++it) {
      const int stage = it % S;
      mbar_wait(&full[stage], (it / S) & 1);
      const uint32_t a_hi = smem_u32(smem + (size_t)stage * Cfg::STAGE) + (uint32_t)(cw * 64 * 128);
      const uint32_t a_lo = a_hi + A_TILE;
      const uint32_t b_hi = smem_u32(smem + (size_t)stage * Cfg::STAGE) + 2 * A_TILE;
      const uint32_t b_lo = b_hi + Cfg::B_TILE;
      wgmma_fence();
      fence_acc(part0);
      mma3_chunk<BN>(part0, a_hi, a_lo, b_hi, b_lo, 0);
      if constexpr (DUAL && !ONE_PART) {
        fence_acc(part1);
        mma3_chunk<BN>(part1, a_hi, a_lo, b_lo + Cfg::B_TILE, b_lo + 2 * Cfg::B_TILE, 0);
      }
      wgmma_commit();
      wgmma_wait_all();
      if constexpr (ONE_PART) {
        fence_acc(part0);
#pragma unroll
        for (int i = 0; i < NA; ++i) acc0[i] += part0[i];
        wgmma_fence();
        fence_acc(part0);
        mma3_chunk<BN>(part0, a_hi, a_lo, b_lo + Cfg::B_TILE, b_lo + 2 * Cfg::B_TILE, 0);
        wgmma_commit();
        wgmma_wait_all();
      }
      if ((tid & 31) == 0) mbar_arrive(&empty[stage]);   // this warp's MMAs have read the stage (and its tile slot)
      fence_acc(part0);
#pragma unroll
      for (int i = 0; i < NA; ++i) (ONE_PART ? acc1 : acc0)[i] += part0[i];
      if constexpr (DUAL && !ONE_PART) {
        fence_acc(part1);
#pragma unroll
        for (int i = 0; i < NA; ++i) acc1[i] += part1[i];
      }
    }

    // the tile's coordinates only now, so that they take no registers beside the accumulators in the loop above
    const int ct = tile % ncol_tiles;
    const long long row0 = (long long)(tile / ncol_tiles) * BM;
    const int col0 = ct * BN;
    // condition broadcast vectors of this tile: qs[s][slot][c] = cond[n_first + s, :] . Wc_slot[:, col0 + c]
    const int n_first = (int)(row0 / p.rows_out);
    if (p.nslots > 0) {
      named_bar_sync(1, CONSUMER_THREADS);    // the previous tile's epilogue has read qs
      for (int o = ctid; o < nqs; o += CONSUMER_THREADS) {
        const int c = o % BN, slot = (o / BN) % p.nslots, s = o / (BN * p.nslots);
        float q = 0.f;
        const int n = n_first + s;
        if (col0 + c < p.ncols && n < p.N) {
          const float* y = p.cond + (size_t)n * p.C;
          const float* wc = p.slot_w[slot] + col0 + c;
          const int ws = p.slot_acc[slot] ? p.terms[p.slot_term[slot]].w2_stride : p.terms[p.slot_term[slot]].w_stride;
          for (int j = 0; j < p.C; ++j) q = fmaf(__ldg(y + j), __ldg(wc + (size_t)j * ws), q);
        }
        qs[o] = q;
      }
      named_bar_sync(1, CONSUMER_THREADS);    // qs complete
    }

    // =========================== epilogue: straight from the accumulator registers ===========================
    // the thread's two rows, h = 0 and 1, each as its own copy of the code: with a loop over h, the accumulators of a
    // wide tile could end up indexed at run time (in local memory)
    auto row_epilogue = [&](auto h_const) {
      constexpr int h = decltype(h_const)::value;
      const int lrow = cw * 64 + frag_row(wt, 2 * h);
      const long long R = row0 + lrow;
      if (R >= p.total_rows) return;
      const int n = (int)(R / p.rows_out), r = (int)(R % p.rows_out);
      const size_t orow = (size_t)R * p.ncols;
      // condition slots, then pass-through terms, into the accumulators in place: each slot or term is a runtime loop
      // around the unrolled columns, so that the accumulators are only ever indexed by constants
      for (int slot = 0; slot < p.nslots; ++slot) {
        const TermDev& tm = p.terms[p.slot_term[slot]];
        const float coef = tm.op.rowsum ? __ldg(tm.op.rowsum + r) : 1.f;
        const float* q = qs + ((size_t)(n - n_first) * p.nslots + slot) * BN + frag_col(wt, 0);
        if (p.slot_acc[slot] == 0) {
#pragma unroll
          for (int g = 0; g < NA / 4; ++g) {
            const int i = 4 * g + 2 * h;
            acc0[i] = fmaf(coef, q[8 * g], acc0[i]); acc0[i + 1] = fmaf(coef, q[8 * g + 1], acc0[i + 1]);
          }
        } else if (DUAL) {
#pragma unroll
          for (int g = 0; g < NA / 4; ++g) {
            const int i = 4 * g + 2 * h;
            acc1[i] = fmaf(coef, q[8 * g], acc1[i]); acc1[i + 1] = fmaf(coef, q[8 * g + 1], acc1[i + 1]);
          }
        }
      }
      if constexpr (PASS) {
        for (int q = p.nterms; q < p.nterms + p.npass; ++q) {   // pass-through terms (F == ncols)
          const TermDev& tm = p.terms[q];
          const float* src = tm.src + (size_t)n * tm.src_rows * tm.src_stride;
#pragma unroll
          for (int g = 0; g < NA / 4; ++g) {
            const int i = 4 * g + 2 * h;
            const int c = col0 + frag_col(wt, i);
            if (c >= p.ncols) continue;
            const float2 s = pass_row2(tm.op, r, src + c, (size_t)tm.src_stride);
            acc0[i] += s.x; acc0[i + 1] += s.y;
          }
        }
      }
      const float* bias_row = (linear && p.bias != nullptr) ? p.bias + (p.bias_per_row ? (size_t)r * p.ncols : 0) : nullptr;
#pragma unroll
      for (int g = 0; g < NA / 4; ++g) {
        const int i = 4 * g + 2 * h;
        const int c = col0 + frag_col(wt, i);
        if (c >= p.ncols) continue;
        float v0[2] = {acc0[i], acc0[i + 1]}, v1[2] = {0.f, 0.f};
        if (DUAL) { v1[0] = acc1[i]; v1[1] = acc1[i + 1]; }
        float o1[2], o2[2];
        bool write2 = false;
        if (linear) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float v = v0[e] + (bias_row != nullptr ? __ldg(bias_row + c + e) : 0.f);
            if (p.act == CAPE_ACT_LEAKY) v = v > 0.f ? v : p.alpha * v;
            else if (p.act == CAPE_ACT_RELU) v = fmaxf(v, 0.f);
            o1[e] = v;
          }
        } else if (p.epilogue == CAPE_EPI_AFFINE) {
          write2 = p.out2 != nullptr;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float rg = fmaxf(v0[e], 0.f);
            o1[e] = (DUAL ? v1[e] : 0.f) + rg;
            o2[e] = rg;
          }
        } else {
          const float2 ax = use_aux ? __ldg(reinterpret_cast<const float2*>(p.aux + orow + c)) : make_float2(0.f, 0.f);
          const float a2[2] = {ax.x, ax.y};
          if (p.epilogue == CAPE_EPI_SLOPE) {
#pragma unroll
            for (int e = 0; e < 2; ++e) o1[e] = v0[e] * (a2[e] > 0.f ? 1.f : p.alpha);
          } else {
            write2 = p.out2 != nullptr;
#pragma unroll
            for (int e = 0; e < 2; ++e) { o1[e] = v0[e]; o2[e] = a2[e] > 0.f ? v0[e] : 0.f; }
          }
        }
        *reinterpret_cast<float2*>(p.out + orow + c) = make_float2(o1[0], o1[1]);
        if (write2) *reinterpret_cast<float2*>(p.out2 + orow + c) = make_float2(o2[0], o2[1]);
      }
    };
    row_epilogue(std::integral_constant<int, 0>{});
    row_epilogue(std::integral_constant<int, 1>{});
  }
}

// cuTensorMapEncodeTiled from the driver the runtime has loaded (the library does not link against libcuda)
PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (fn == nullptr) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
  }
  return fn;
}

// wT (row c at wT + c * stride, F valid k) as a [ncols x F] tensor in boxes of 32 k x BN columns
int encode_weight_map(CUtensorMap* m, const float* wT, int F, int stride, int ncols, int bn) {
  const auto encode = tensor_map_encoder();
  if (encode == nullptr) {
    set_error("conv_wg_kernel: cuTensorMapEncodeTiled is not available from the CUDA driver");
    return -2;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)F, (cuuint64_t)ncols};
  const cuuint64_t strides[1] = {(cuuint64_t)stride * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)bn};
  const cuuint32_t estrides[2] = {1, 1};
  const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(wT), dims, strides, box, estrides,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("conv_wg_kernel: cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return -2;
  }
  return 0;
}

template <int BN, bool DUAL, bool PASS = false>
int launch_conv(const cape_topology* t, const ConvParams& p, cudaStream_t st) {
  using Cfg = ConvCfg<BN, DUAL>;
  WeightMaps maps;
  memset(&maps, 0, sizeof(maps));
  for (int i = 0; i < p.nterms; ++i) {
    const TermDev& tm = p.terms[i];
    if (encode_weight_map(&maps.w[i][0], tm.wT, tm.F, tm.wT_stride, p.ncols, BN) != 0) return -2;
    if (DUAL && tm.w2T != nullptr &&
        encode_weight_map(&maps.w[i][1], tm.w2T, tm.F, tm.w2T_stride, p.ncols, BN) != 0)
      return -2;
  }
  int nqs = 0;
  if (p.nslots > 0) {
    const long long rlast_max = BM - 1;
    const int S = (int)(rlast_max / p.rows_out) + 2;
    nqs = S * p.nslots * BN;
  }
  const int smem = 1024 + Cfg::RING + BAR_BYTES + nqs * 4;
  static bool configured = false;
  if (!configured) {
    CAPE_CHECK_CUDA(cudaFuncSetAttribute(conv_wg_kernel<BN, DUAL, PASS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         1024 + Cfg::RING + BAR_BYTES + QS_MAX_FLOATS * 4));
    configured = true;
  }
  // tiles numbered with the column tiles fastest; one persistent CTA per SM (or per tile, if fewer)
  const int ncol_tiles = (p.ncols + BN - 1) / BN;
  const long long ntiles = (p.total_rows + BM - 1) / BM * ncol_tiles;
  if (ntiles + t->sm_count >= (1LL << 31)) {
    set_error("conv_wg_kernel: too many tiles");
    return -1;
  }
  const int grid = (int)std::min<long long>(ntiles, t->sm_count);
  conv_wg_kernel<BN, DUAL, PASS><<<grid, CONV_THREADS, smem, st>>>(p, maps, nqs, ncol_tiles, (int)ntiles,
                                                                   t->tile_counter);
  CAPE_CHECK_CUDA(cudaGetLastError());
  count_launches(1);
  return 1;
}

// column tile width: the whole output row up to 128 columns (64 with two accumulators), so that the running sums and
// the chunk accumulators fit the registers
int pick_bn(int ncols, bool dual) {
  if (ncols <= 32) return 32;
  if (ncols <= 64 || dual) return 64;
  return 128;
}

// false if the condition vectors of a tile would not fit the staging buffer
bool qs_fits(const ConvParams& p, int bn) {
  if (p.nslots == 0) return true;
  const long long max_samples = (BM - 1) / p.rows_out + 2;
  return max_samples * p.nslots * bn <= QS_MAX_FLOATS;
}

}  // namespace

static bool g_tc_enabled = true;
int g_tuning[32] = {0};   // experiment knobs (cape_set_tuning), see ellconv_params.cuh
bool tensor_cores_enabled() { return g_tc_enabled; }

int launch_ellconv_tc(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st) {
  if (!g_tc_enabled) return 0;
  if (p.ncols % 32 != 0 || p.ncols < 32 || !p.ovec) return 0;
  if ((dual ? 2 : 1) * p.ncols > 512) return 0;
  long long kred = 0;
  for (int i = 0; i < p.nterms; ++i) {
    const TermDev& tm = p.terms[i];
    if (!tm.vec || tm.wT == nullptr || (tm.wT_stride % 4) != 0 || !aligned16(tm.wT)) return 0;
    if (tm.w2 != nullptr && (tm.w2T == nullptr || (tm.w2T_stride % 4) != 0 || !aligned16(tm.w2T))) return 0;
    if (tm.stash != nullptr && (tm.stash_stride % 4) != 0) return 0;
    kred += tm.F;
  }
  for (int i = p.nterms; i < p.nterms + p.npass; ++i)   // pass-through terms: float2 loads in the epilogue
    if (!p.terms[i].vec) return 0;
  if (kred < 64) return 0;                       // tiny reductions: the SIMT kernel is as good and simpler
  const int bn = pick_bn(p.ncols, dual);
  if (!qs_fits(p, bn)) return 0;
  if (p.npass > 0) {                             // the encoder's residual blocks: single accumulator
    if (dual) return 0;
    if (bn == 32) return launch_conv<32, false, true>(t, p, st);
    if (bn == 64) return launch_conv<64, false, true>(t, p, st);
    return launch_conv<128, false, true>(t, p, st);
  }
  if (dual) return bn == 32 ? launch_conv<32, true>(t, p, st) : launch_conv<64, true>(t, p, st);
  if (bn == 32) return launch_conv<32, false>(t, p, st);
  if (bn == 64) return launch_conv<64, false>(t, p, st);
  return launch_conv<128, false>(t, p, st);
}

// all-plain-operand calls: 1 = launched, 0 = not eligible (the caller falls through to the gather kernels)
int launch_gemm_tc(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st) {
  if (!tensor_cores_enabled() || g_tuning[8] == 1) return 0;
  if (dual || p.epilogue == CAPE_EPI_AFFINE || p.npass > 0) return 0;
  if (p.ncols % 16 != 0 || p.ncols < 32 || !p.ovec) return 0;
  if (p.total_rows >= (1LL << 31)) return 0;
  long long kred = 0;
  for (int i = 0; i < p.nterms; ++i) {
    const TermDev& tm = p.terms[i];
    if (tm.op.idx != nullptr || tm.src_rows != p.rows_out || !tm.vec || tm.stash != nullptr) return 0;
    if (tm.wT == nullptr || (tm.wT_stride % 4) != 0 || !aligned16(tm.wT)) return 0;
    kred += tm.F;
  }
  if (kred < 32) return 0;
  for (int s = 0; s < p.nslots; ++s)
    if (p.slot_acc[s] != 0) return 0;
  const int bn = pick_bn(p.ncols, false);
  if (!qs_fits(p, bn)) return 0;
  if (bn == 32) return launch_conv<32, false>(t, p, st);
  if (bn == 64) return launch_conv<64, false>(t, p, st);
  return launch_conv<128, false>(t, p, st);
}

}  // namespace cape

extern "C" int cape_set_tuning(int key, int value) {
  if (key < 0 || key >= 32) return -1;
  const int prev = cape::g_tuning[key];
  cape::g_tuning[key] = value;
  return prev;
}

extern "C" int cape_tensor_cores_enabled(void) { return cape::g_tc_enabled ? 1 : 0; }

extern "C" int cape_set_tensor_cores(int enable) {
  const int prev = cape::g_tc_enabled ? 1 : 0;
  cape::g_tc_enabled = enable != 0;
  return prev;
}
