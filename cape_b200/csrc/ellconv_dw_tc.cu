// Tensor-core (wgmma, sm_90a) weight-gradient kernel:  dW[f, c] = sum_{n,v} A[n,v,f] * G[n,v,c]   (3xTF32, fp32
// accumulation), for gathered basis operands (A = op . X) and plain ones (A = X) alike.
//
// The reduction runs over the rows (up to N*6890), so rows are the MMA K dimension.  wgmma reads 32-bit operands
// K-major only, so the producers transpose on the way into shared memory: a warp loads 16 rows of the chunk, two
// adjacent float4 (32 bytes, one full sector) of each, and each lane writes its four values into four tile rows at
// the column of its row -- in the swizzled layout the 32 lanes of one such store hit 32 different banks.  A CTA owns
// a 128-wide slice of f, a BN-wide slice of the output columns and one split of the rows, and runs its warpgroups
// around a ring of shared-memory stages (32 rows each):
//  - the producer warpgroups (two up to BN = 128, one at BN = 256) take alternate chunks: each thread issues all of its
//    chunk's loads (8 float4 of A, BN / 16 of G), then waits for the stage to be free, splits the values into hi/lo,
//    stores them transposed and arrives on the stage's `full` mbarrier.  A whole chunk per warpgroup keeps twice as
//    many loads in flight per thread as sharing each chunk would: the loads are latency-bound.  At BN = 256 the 128
//    accumulators of a consumer thread need more than the 128 registers a 512-thread CTA allows, so that CTA has 384
//    threads, and its ring only two stages: the producer loads its next chunk into registers while it waits for the
//    stage;
//  - the last two warpgroups, the consumers, each own 64 f rows: wait on `full`, issue the chunk's 12 MMAs into the
//    running accumulator, then wait until only this chunk's MMAs are pending (wgmma.wait_group 1) and release the
//    previous chunk's stage on its `empty` mbarrier.  The tensor pipe does not drain between chunks.
// setmaxnreg moves registers from the producers to the consumers, which hold the accumulators.  The grid is 1-D with
// the column tiles and then the f tiles fastest, so the CTAs of one row split run together and read its A and G rows
// from L2 rather than from HBM once per tile.
//
// The tensor core's fp32 accumulation truncates, so a sum over a long chain of MMAs shrinks a little with every MMA;
// the rows per split grow with the batch (the split plan keeps the number of CTAs fixed).  So every DW_FLUSH_CHUNKS
// chunks (2048 rows, more than any split of the batch-64 step has) the consumers wait for their MMAs, add the
// accumulators into the CTA's own output slice in fp32 (red.global: no round trip, no registers; the first flush
// stores unless it accumulates into dW) and start the next chunk with scale_d = 0.  Each element has one owning
// thread, so the order of the adds is fixed.  Partial sums of the row splits go to the topology workspace and are
// reduced deterministically (reduce_splits_kernel).
#include "common.cuh"
#include "ellconv_params.cuh"
#include "tc_common.cuh"

namespace cape {

namespace {

using namespace tc;

constexpr int DW_KCH = 32;                   // rows (K) per chunk
constexpr int DW_A_TILE = 128 * 128;         // 128 f x 32 rows, hi or lo
constexpr int DW_BAR_BYTES = 256;            // the ring's mbarriers
constexpr int DW_SMEM_MAX = 227 * 1024;      // dynamic shared memory per CTA on sm_90
constexpr int DW_FLUSH_CHUNKS = 64;          // chunks (2048 rows) per MMA chain, unless set by cape_set_tuning(11, .)

struct DwTcParams {
  int rows_out, ncols, F, src_rows, src_stride;
  long long total_rows, rows_per_split;
  const float* src;
  OpView op;
  const float* g;
  float* out;          // dw (nsplit == 1) or workspace [nsplit, F, ncols]
  long long out_rs;
  int nsplit, accumulate;
  int ftiles, ctiles;
  int flush_chunks;    // chunks per MMA chain: the consumers add their accumulators into `out` every flush_chunks
};

template <int BN>
struct DwCfg {
  static constexpr int G_TILE = BN * 128;
  static constexpr int STAGE = 2 * DW_A_TILE + 2 * G_TILE;
  // 5 stages at BN = 32, 4 at 64, 3 at 128, 2 at 256
  static constexpr int STAGES = (DW_SMEM_MAX - 1024 - DW_BAR_BYTES) / STAGE;
  static constexpr int RING = STAGES * STAGE;
  static constexpr int SMEM_BYTES = 1024 + RING + DW_BAR_BYTES;
  static constexpr int PRODUCERS = BN <= 128 ? 2 : 1;             // producer warpgroups
  static constexpr int THREADS = 128 * (PRODUCERS + 2);
  // per-thread registers after setmaxnreg: PRODUCERS * PRODUCER_REGS + 2 * CONSUMER_REGS <= (PRODUCERS + 2) * (the
  // launch limit of 65536 / THREADS, rounded down to 8)
  static constexpr int PRODUCER_REGS = BN <= 128 ? 120 : 152;
  static constexpr int CONSUMER_REGS = BN <= 128 ? 136 : 176;
  static_assert(PRODUCERS * PRODUCER_REGS + 2 * CONSUMER_REGS <= (PRODUCERS + 2) * (65536 / THREADS / 8 * 8),
                "register split exceeds the launch budget");
  static_assert(STAGES >= 2, "the ring needs at least two stages");
  static_assert(2 * STAGES * 8 <= DW_BAR_BYTES, "mbarrier area too small");
};

// *o += v in fp32 (round to nearest) by the L2, without a round trip to the issuing thread (red.global)
__device__ __forceinline__ void red_add(float* o, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(__cvta_generic_to_global(o)), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add2(float* o, float v0, float v1) {     // o 8-byte aligned
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(__cvta_generic_to_global(o)), "f"(v0), "f"(v1)
               : "memory");
}

template <int BN, bool CHAINS>
__global__ void __launch_bounds__(DwCfg<BN>::THREADS, 1) dw_wg_kernel(const __grid_constant__ DwTcParams p) {
  using Cfg = DwCfg<BN>;
  constexpr int S = Cfg::STAGES;
  constexpr int NA = BN / 2;
  constexpr int GQ = BN / 16;                // float4 column groups of G per producer thread
  extern __shared__ uint8_t smem_raw[];
  char* smem = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::RING);
  uint64_t* empty = full + S;

  const int tid = threadIdx.x, wgi = tid >> 7, lane = tid & 31;
  const int ct = (int)(blockIdx.x % (unsigned)p.ctiles);
  const int ft = (int)(blockIdx.x / (unsigned)p.ctiles % (unsigned)p.ftiles);
  const int split = (int)(blockIdx.x / (unsigned)(p.ctiles * p.ftiles));
  const int ftile = ft * 128;
  const int col0 = ct * BN;
  const long long rbeg = (long long)split * p.rows_per_split;
  const long long rend = min(p.total_rows, rbeg + p.rows_per_split);
  const long long nchunks = (rend - rbeg + DW_KCH - 1) / DW_KCH;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 128);              // every thread of the chunk's producer warpgroup
      mbar_init(&empty[s], 8);               // one lane per consumer warp
    }
  }
  __syncthreads();

  if (wgi < Cfg::PRODUCERS) {
    // ==================== producers: warpgroup wgi loads chunks wgi, wgi + PRODUCERS, ... ====================
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    // warp w4 of the warpgroup: rows 16 (w4 & 1) .. + 15 of the chunk, one per lane pair; float4 groups g0 + 4 i with
    // g0 = 2 (w4 >> 1) + (lane & 1), so a load instruction reads 32 contiguous bytes of each of its 16 rows
    const int w4 = (tid >> 5) & 3;
    const int kr = 16 * (w4 & 1) + (lane >> 1), g0 = 2 * (w4 >> 1) + (lane & 1);
    // tile rows 4 (g0 + 4 i) + e for i = 0, 1, ... lie 16 i rows (2048 bytes) apart with the same swizzle
    uint32_t off[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) off[e] = sw_off(4 * g0 + e, kr);
    for (long long kc = wgi; kc < nchunks; kc += Cfg::PRODUCERS) {
      const int R = (int)(rbeg + kc * DW_KCH) + kr;     // rows < 2^31 (launch_ellconv_dw_tc)
      const bool live = R < rend;
      const int Q = live ? R : (int)rbeg;
      const int n = Q / p.rows_out, r = Q % p.rows_out;
      const float* base = p.src + (size_t)n * p.src_rows * p.src_stride;
      float4 ra[8], rg[GQ];
#pragma unroll
      for (int i = 0; i < GQ; ++i) {
        const int c = col0 + 4 * (g0 + 4 * i);
        rg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live && c < p.ncols) rg[i] = ldg4(p.g + (size_t)R * p.ncols + c);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int f = ftile + 4 * (g0 + 4 * i);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live && f < p.F) {
          if (p.op.idx == nullptr) v = ldg4(base + (size_t)r * p.src_stride + f);
          else ell_gather4(p.op, r, base + f, (size_t)p.src_stride, v);
        }
        ra[i] = v;
      }
      const int stage = (int)(kc % S);
      mbar_wait(&empty[stage], (uint32_t)((kc / S) & 1) ^ 1);
      char* a_hi = smem + (size_t)stage * Cfg::STAGE;
      char* a_lo = a_hi + DW_A_TILE;
      char* g_hi = a_lo + DW_A_TILE;
      char* g_lo = g_hi + Cfg::G_TILE;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        char* hi = a_hi + 2048 * i;
        char* lo = a_lo + 2048 * i;
        split_store1(ra[i].x, hi, lo, off[0]);
        split_store1(ra[i].y, hi, lo, off[1]);
        split_store1(ra[i].z, hi, lo, off[2]);
        split_store1(ra[i].w, hi, lo, off[3]);
      }
#pragma unroll
      for (int i = 0; i < GQ; ++i) {
        char* hi = g_hi + 2048 * i;
        char* lo = g_lo + 2048 * i;
        split_store1(rg[i].x, hi, lo, off[0]);
        split_store1(rg[i].y, hi, lo, off[1]);
        split_store1(rg[i].z, hi, lo, off[2]);
        split_store1(rg[i].w, hi, lo, off[3]);
      }
      fence_proxy_async();                   // generic-proxy smem writes -> visible to the tensor core's (async) proxy
      mbar_arrive(&full[stage]);
    }
    return;
  }

  // =========================== consumers ===========================
  setmaxnreg_inc<Cfg::CONSUMER_REGS>();
  const int cw = wgi - Cfg::PRODUCERS, wt = tid & 127;
  float* out = p.out + (p.nsplit > 1 ? (size_t)split * p.F * p.out_rs : 0);
  const bool vec2 = (p.out_rs % 2 == 0) && ((reinterpret_cast<uintptr_t>(out) & 7u) == 0);
  float acc[NA];
#pragma unroll
  for (int i = 0; i < NA; ++i) acc[i] = 0.f;
  fence_acc(acc);
  if constexpr (!CHAINS) {
    // ---- every split fits one chain: one pass, then the accumulators -> dW or the split's partial sums ----
    for (long long kc = 0; kc < nchunks; ++kc) {
      const int stage = (int)(kc % S);
      mbar_wait(&full[stage], (uint32_t)((kc / S) & 1));
      const uint32_t base = smem_u32(smem + (size_t)stage * Cfg::STAGE);
      const uint32_t a_hi = base + (uint32_t)(cw * 64 * 128), a_lo = a_hi + DW_A_TILE;
      const uint32_t g_hi = base + 2 * DW_A_TILE, g_lo = g_hi + Cfg::G_TILE;
      wgmma_fence();
      mma3_chunk<BN>(acc, a_hi, a_lo, g_hi, g_lo, 1);
      wgmma_commit();
      wgmma_wait<1>();                       // the previous chunk's MMAs have read their stage
      if (kc > 0 && lane == 0) mbar_arrive(&empty[(int)((kc - 1) % S)]);
    }
    wgmma_wait<0>();
    fence_acc(acc);
#pragma unroll
    for (int i = 0; i < NA; i += 2) {
      const int f = ftile + cw * 64 + frag_row(wt, i);
      const int c = col0 + frag_col(wt, i);
      if (f >= p.F || c >= p.ncols) continue;
      float* o = out + (size_t)f * p.out_rs + c;
      if (p.nsplit == 1 && p.accumulate) {
        o[0] += acc[i];
        o[1] += acc[i + 1];
      } else if (vec2) {
        *reinterpret_cast<float2*>(o) = make_float2(acc[i], acc[i + 1]);
      } else {
        o[0] = acc[i];
        o[1] = acc[i + 1];
      }
    }
  } else {
    // ---- chains of flush_chunks chunks: after each, the accumulators are stored into this CTA's slice of dW or of
    // the split's partial sums (added into dW when accumulating) the first time and added in fp32 after that.  Each
    // element has one owning thread, whose adds follow program order.
    bool flushed = false;
    auto flush = [&]() {
      const bool add = flushed || (p.nsplit == 1 && p.accumulate);
      // opaque to the compiler: the addresses are computed here, not kept live across the loop (no spare registers)
      float* dst = out;
      int t = wt;
      asm volatile("" : "+l"(dst), "+r"(t));
#pragma unroll
      for (int i = 0; i < NA; i += 2) {
        const int f = ftile + cw * 64 + frag_row(t, i);
        const int c = col0 + frag_col(t, i);
        if (f >= p.F || c >= p.ncols) continue;
        float* o = dst + (size_t)f * p.out_rs + c;
        if (add && vec2) {
          red_add2(o, acc[i], acc[i + 1]);
        } else if (add) {
          red_add(o, acc[i]);
          red_add(o + 1, acc[i + 1]);
        } else if (vec2) {
          *reinterpret_cast<float2*>(o) = make_float2(acc[i], acc[i + 1]);
        } else {
          o[0] = acc[i];
          o[1] = acc[i + 1];
        }
      }
      flushed = true;
    };
    for (long long k0 = 0; k0 < nchunks; k0 += p.flush_chunks) {
      const long long k1 = min(nchunks, k0 + p.flush_chunks);
      for (long long kc = k0; kc < k1; ++kc) {
        const int stage = (int)(kc % S);
        mbar_wait(&full[stage], (uint32_t)((kc / S) & 1));
        const uint32_t base = smem_u32(smem + (size_t)stage * Cfg::STAGE);
        const uint32_t a_hi = base + (uint32_t)(cw * 64 * 128), a_lo = a_hi + DW_A_TILE;
        const uint32_t g_hi = base + 2 * DW_A_TILE, g_lo = g_hi + Cfg::G_TILE;
        wgmma_fence();
        mma3_chunk<BN>(acc, a_hi, a_lo, g_hi, g_lo, kc == k0 ? 0 : 1);
        wgmma_commit();
        wgmma_wait<1>();
        if (kc > 0 && lane == 0) mbar_arrive(&empty[(int)((kc - 1) % S)]);
      }
      wgmma_wait<0>();
      fence_acc(acc);
      flush();
    }
  }
}

template <int BN, bool CHAINS>
int launch_dw(const DwTcParams& p, cudaStream_t st) {
  using Cfg = DwCfg<BN>;
  static bool configured = false;
  if (!configured) {
    CAPE_CHECK_CUDA(cudaFuncSetAttribute(dw_wg_kernel<BN, CHAINS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES));
    configured = true;
  }
  const long long nblocks = (long long)p.ftiles * p.ctiles * p.nsplit;
  if (nblocks >= (1LL << 31)) {
    set_error("dw_wg_kernel: too many tiles");
    return -1;
  }
  dw_wg_kernel<BN, CHAINS><<<(unsigned)nblocks, Cfg::THREADS, Cfg::SMEM_BYTES, st>>>(p);
  CAPE_CHECK_CUDA(cudaGetLastError());
  count_launches(1);
  return 1;
}

template <int BN>
int launch_dw(const DwTcParams& p, cudaStream_t st) {
  return p.rows_per_split / DW_KCH > p.flush_chunks ? launch_dw<BN, true>(p, st) : launch_dw<BN, false>(p, st);
}

}  // namespace

// returns 1 if launched (partials in workspace when *nsplit_out > 1), 0 if not eligible, <0 on error
int launch_ellconv_dw_tc(const cape_topology* t, const cape_dw_args* a, const OpView& op, int* nsplit_out,
                         cudaStream_t st) {
  if (!tensor_cores_enabled()) return 0;
  if (a->ncols % 32 != 0 || a->ncols < 32 || a->ncols > 512) return 0;
  if (a->F % 4 != 0 || a->F < 32 || a->src_stride % 4 != 0 || !aligned16(a->src) || !aligned16(a->g)) return 0;
  DwTcParams p{};
  p.rows_out = a->rows_out; p.ncols = a->ncols; p.F = a->F; p.src_rows = a->src_rows; p.src_stride = a->src_stride;
  p.total_rows = (long long)a->N * a->rows_out;
  if (p.total_rows < 4096 || p.total_rows >= (1LL << 31)) return 0;
  p.src = a->src; p.op = op; p.g = a->g;
  const int BN = a->ncols <= 32 ? 32 : (a->ncols <= 64 ? 64 : (a->ncols <= 128 ? 128 : 256));
  p.ftiles = (a->F + 127) / 128;
  p.ctiles = (a->ncols + BN - 1) / BN;
  // about two waves of CTAs over the row splits
  long long nsplit = (2LL * t->sm_count + p.ftiles * p.ctiles - 1) / (p.ftiles * p.ctiles);
  const long long max_by_rows = (p.total_rows + 511) / 512;
  if (nsplit > max_by_rows) nsplit = max_by_rows;
  const long long per = (long long)a->F * a->ncols * (long long)sizeof(float);
  if (nsplit > 1 && nsplit * per > t->workspace_bytes) nsplit = t->workspace_bytes / per;
  if (nsplit < 1) nsplit = 1;
  long long rps = (p.total_rows + nsplit - 1) / nsplit;
  rps = (rps + DW_KCH - 1) / DW_KCH * DW_KCH;
  nsplit = (p.total_rows + rps - 1) / rps;
  p.rows_per_split = rps; p.nsplit = (int)nsplit; p.accumulate = a->accumulate;
  p.flush_chunks = g_tuning[11] > 0 ? g_tuning[11] : (g_tuning[11] < 0 ? INT_MAX : DW_FLUSH_CHUNKS);
  if (nsplit == 1) { p.out = a->dw; p.out_rs = a->dw_stride; }
  else { p.out = (float*)t->workspace; p.out_rs = a->ncols; }
  *nsplit_out = (int)nsplit;
  if (BN == 32) return launch_dw<32>(p, st);
  if (BN == 64) return launch_dw<64>(p, st);
  if (BN == 128) return launch_dw<128>(p, st);
  return launch_dw<256>(p, st);
}

}  // namespace cape
