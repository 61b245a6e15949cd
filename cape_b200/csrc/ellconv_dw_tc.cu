// Tensor-core (wgmma, sm_90a) weight-gradient kernel:  dW[f, c] = sum_{n,v} A[n,v,f] * G[n,v,c]   (3xTF32, fp32
// accumulation), for gathered basis operands (A = op . X) and plain ones (A = X) alike.
//
// The reduction runs over the rows (up to N*6890), so rows are the MMA K dimension.  wgmma reads 32-bit operands
// K-major only, so the producers transpose on the way into shared memory: lane k of a warp loads row k of the chunk
// (a float4 of four consecutive f, or c for G) and writes the four values into four tile rows at column k -- in the
// swizzled layout the 32 lanes of one such store hit 32 different banks.  One CTA (two warpgroups, 64 f each) owns a
// 128-wide slice of f, a BN-wide slice of the output columns and one split of the rows; the chunks are
// double-buffered as in ellconv_tc.cu.  Partial sums of the row splits go to the topology workspace and are reduced
// deterministically (reduce_splits_kernel).
#include "common.cuh"
#include "ellconv_params.cuh"
#include "tc_common.cuh"

namespace cape {

namespace {

using namespace tc;

constexpr int DW_THREADS = 256;
constexpr int DW_KCH = 32;                   // rows (K) per chunk
constexpr int DW_A_TILE = 128 * 128;         // 128 f x 32 rows, hi or lo

struct DwTcParams {
  int rows_out, ncols, F, src_rows, src_stride;
  long long total_rows, rows_per_split;
  const float* src;
  OpView op;
  const float* g;
  float* out;          // dw (nsplit == 1) or workspace [nsplit, F, ncols]
  long long out_rs;
  int nsplit, accumulate;
};

template <int BN>
struct DwCfg {
  static constexpr int G_TILE = BN * 128;
  static constexpr int STAGE = 2 * DW_A_TILE + 2 * G_TILE;
  static constexpr int SMEM_BYTES = 1024 + 2 * STAGE;
};

template <int BN>
__global__ void __launch_bounds__(DW_THREADS, BN <= 64 ? 2 : 1) dw_wg_kernel(const __grid_constant__ DwTcParams p) {
  using Cfg = DwCfg<BN>;
  constexpr int NA = BN / 2;
  constexpr int GQ = BN / 32;                // float4 column groups of G per thread
  extern __shared__ uint8_t smem_raw[];
  char* smem = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = tid >> 7, wt = tid & 127;
  const int ftile = blockIdx.x * 128;
  const int col0 = blockIdx.z * BN;
  const long long rbeg = (long long)blockIdx.y * p.rows_per_split;
  const long long rend = min(p.total_rows, rbeg + p.rows_per_split);
  const long long nchunks = (rend - rbeg + DW_KCH - 1) / DW_KCH;

  float4 ra[4], rg[GQ];
  // lane = row of the chunk; warp w covers the float4 groups w, w + 8, ... of f (A) and of c (G)
  auto load_chunk = [&](long long kc) {
    const long long R = rbeg + kc * DW_KCH + lane;
    const bool live = R < rend;
    const long long Q = live ? R : rbeg;
    const int n = (int)(Q / p.rows_out), r = (int)(Q % p.rows_out);
    const float* base = p.src + (size_t)n * p.src_rows * p.src_stride;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = ftile + 4 * (warp + 8 * i);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (live && f < p.F) {
        if (p.op.idx == nullptr) v = ldg4(base + (size_t)r * p.src_stride + f);
        else ell_gather4(p.op, r, base + f, (size_t)p.src_stride, v);
      }
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < GQ; ++i) {
      const int c = col0 + 4 * (warp + 8 * i);
      rg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (live && c < p.ncols) rg[i] = ldg4(p.g + (size_t)R * p.ncols + c);
    }
  };
  auto store_chunk = [&](int stage) {
    char* a_hi = smem + (size_t)stage * Cfg::STAGE;
    char* a_lo = a_hi + DW_A_TILE;
    char* g_hi = a_lo + DW_A_TILE;
    char* g_lo = g_hi + Cfg::G_TILE;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = 4 * (warp + 8 * i);
      split_store1(ra[i].x, a_hi, a_lo, sw_off(m, lane));
      split_store1(ra[i].y, a_hi, a_lo, sw_off(m + 1, lane));
      split_store1(ra[i].z, a_hi, a_lo, sw_off(m + 2, lane));
      split_store1(ra[i].w, a_hi, a_lo, sw_off(m + 3, lane));
    }
#pragma unroll
    for (int i = 0; i < GQ; ++i) {
      const int m = 4 * (warp + 8 * i);
      split_store1(rg[i].x, g_hi, g_lo, sw_off(m, lane));
      split_store1(rg[i].y, g_hi, g_lo, sw_off(m + 1, lane));
      split_store1(rg[i].z, g_hi, g_lo, sw_off(m + 2, lane));
      split_store1(rg[i].w, g_hi, g_lo, sw_off(m + 3, lane));
    }
  };

  float acc[NA];
#pragma unroll
  for (int i = 0; i < NA; ++i) acc[i] = 0.f;

  if (nchunks > 0) {
    load_chunk(0);
    store_chunk(0);
    fence_proxy_async();
    __syncthreads();
    for (long long kc = 0;; ++kc) {
      const int stage = (int)(kc & 1);
      const uint32_t base = smem_u32(smem + (size_t)stage * Cfg::STAGE);
      const uint32_t a_hi = base + (uint32_t)(wgi * 64 * 128), a_lo = a_hi + DW_A_TILE;
      const uint32_t g_hi = base + 2 * DW_A_TILE, g_lo = g_hi + Cfg::G_TILE;
      wgmma_fence();
      fence_acc(acc);
      mma3_chunk<BN>(acc, a_hi, a_lo, g_hi, g_lo, 1);
      wgmma_commit();
      const bool more = kc + 1 < nchunks;
      if (more) {
        load_chunk(kc + 1);
        store_chunk(stage ^ 1);
      }
      wgmma_wait_all();
      fence_acc(acc);
      if (!more) break;
      fence_proxy_async();
      __syncthreads();
    }
  }

  // =========================== epilogue: accumulators -> dW or the split's partial sums ===========================
  float* out = p.out + (p.nsplit > 1 ? (size_t)blockIdx.y * p.F * p.out_rs : 0);
  const bool vec2 = (p.out_rs % 2 == 0) && ((reinterpret_cast<uintptr_t>(out) & 7u) == 0);
#pragma unroll
  for (int i = 0; i < NA; i += 2) {
    const int f = ftile + wgi * 64 + frag_row(wt, i);
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
}

template <int BN>
int launch_dw(const DwTcParams& p, int ftiles, cudaStream_t st) {
  using Cfg = DwCfg<BN>;
  static bool configured = false;
  if (!configured) {
    CAPE_CHECK_CUDA(cudaFuncSetAttribute(dw_wg_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    configured = true;
  }
  dim3 grid(ftiles, p.nsplit, (p.ncols + BN - 1) / BN);
  dw_wg_kernel<BN><<<grid, DW_THREADS, Cfg::SMEM_BYTES, st>>>(p);
  CAPE_CHECK_CUDA(cudaGetLastError());
  count_launches(1);
  return 1;
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
  const int ftiles = (a->F + 127) / 128, ctiles = (a->ncols + BN - 1) / BN;
  // about two waves of CTAs over the row splits
  long long nsplit = (2LL * t->sm_count + ftiles * ctiles - 1) / (ftiles * ctiles);
  const long long max_by_rows = (p.total_rows + 511) / 512;
  if (nsplit > max_by_rows) nsplit = max_by_rows;
  const long long per = (long long)a->F * a->ncols * (long long)sizeof(float);
  if (nsplit > 1 && nsplit * per > t->workspace_bytes) nsplit = t->workspace_bytes / per;
  if (nsplit < 1) nsplit = 1;
  long long rps = (p.total_rows + nsplit - 1) / nsplit;
  rps = (rps + DW_KCH - 1) / DW_KCH * DW_KCH;
  nsplit = (p.total_rows + rps - 1) / rps;
  p.rows_per_split = rps; p.nsplit = (int)nsplit; p.accumulate = a->accumulate;
  if (nsplit == 1) { p.out = a->dw; p.out_rs = a->dw_stride; }
  else { p.out = (float*)t->workspace; p.out_rs = a->ncols; }
  *nsplit_out = (int)nsplit;
  if (BN == 32) return launch_dw<32>(p, ftiles, st);
  if (BN == 64) return launch_dw<64>(p, ftiles, st);
  if (BN == 128) return launch_dw<128>(p, ftiles, st);
  return launch_dw<256>(p, ftiles, st);
}

}  // namespace cape
