// Tensor-core (wgmma, sm_90a) version of the fused ELL-gather Chebyshev convolution, and of the same contraction for
// calls whose terms are all plain tensors (identity operators: 1x1 convs, the split convolution forms, the GroupNorm
// blocks' linear layers).
//
// Same math and epilogues as ellconv.cu, but the [128 x Fin*K] x [Fin*K x BN] contraction runs on the tensor cores
// with fp32 accuracy by 3xTF32 error compensation:  a = a_hi + a_lo (a_hi = top 19 bits, a_lo = the exact remainder),
// acc += a_hi*b_hi + a_lo*b_hi + a_hi*b_lo with fp32 accumulation; the dropped a_lo*b_lo term is ~2^-22 relative.
//
// A CTA of two warpgroups owns one 128-row x BN-column output tile (grid.y walks the column tiles).  All 256 threads
// gather the Chebyshev-basis chunk A[128 rows x 32 k] from neighbour rows (float4 loads, same ELL tables as the SIMT
// path) and load the weight chunk B[BN x 32 k] (K-major copy of W), split both into hi/lo and store them in the
// swizzled K-major layout; each warpgroup then issues wgmma m64nBNk8 for its 64 rows.  The shared-memory tiles are
// double-buffered: the loads of chunk j+1 are in flight while the MMAs of chunk j run.
//
// Every chunk's products go to a fresh register accumulator that is added to the running sum in fp32 with
// round-to-nearest, so the tensor core's truncating accumulation chain is one chunk (12 MMAs) long instead of the whole
// reduction: long reductions would otherwise drift from the fp64 truth by more than 1e-4 (cape_conv_args.precise
// has no effect).
#include "common.cuh"
#include "ellconv_params.cuh"
#include "tc_common.cuh"

namespace cape {

namespace {

using namespace tc;

constexpr int WG_THREADS = 256;
constexpr int A_TILE = BM * 128;              // 128 rows x 32 fp32
constexpr int QS_MAX_FLOATS = 8192;           // condition vectors of the tile's samples and columns

template <int BN, bool DUAL>
struct ConvCfg {
  static constexpr int B_TILE = BN * 128;
  static constexpr int STAGE = 2 * A_TILE + (DUAL ? 4 : 2) * B_TILE;
  static constexpr int RING = 2 * STAGE;
};

template <int BN, bool DUAL>
__global__ void __launch_bounds__(WG_THREADS, BN <= 32 && !DUAL ? 2 : 1) conv_wg_kernel(const __grid_constant__ ConvParams p, int nqs) {
  using Cfg = ConvCfg<BN, DUAL>;
  constexpr int NA = BN / 2;                  // accumulator registers per thread
  extern __shared__ uint8_t smem_raw[];
  char* smem = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* qs = reinterpret_cast<float*>(smem + Cfg::RING);

  const int tid = threadIdx.x, wgi = tid >> 7, wt = tid & 127;
  const long long row0 = (long long)blockIdx.x * BM;
  const int col0 = blockIdx.y * BN;
  const int n_first = (int)(row0 / p.rows_out);

  // condition broadcast vectors of this tile: qs[s][slot][c] = cond[n_first + s, :] . Wc_slot[:, col0 + c]
  if (p.nslots > 0) {
    for (int o = tid; o < nqs; o += WG_THREADS) {
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
  }

  // producer mapping: 8 threads per 128-byte tile row (one float4 of k each), 32 row slots
  const int l8 = tid & 7, rs = tid >> 3;
  int rn[4], rr[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long R = row0 + rs + 32 * i;
    if (R < p.total_rows) { rn[i] = (int)(R / p.rows_out); rr[i] = (int)(R % p.rows_out); }
    else { rn[i] = -1; rr[i] = 0; }
  }
  const bool do_stash = blockIdx.y == 0;      // one column tile writes the basis copies

  float4 ra[4], rb[BN / 32], rb2[DUAL ? BN / 32 : 1];

  auto load_chunk = [&](int t, int f0) {
    const TermDev& tm = p.terms[t];
    const int f = f0 + l8 * 4;
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < tm.F) {
        // invalid (beyond-the-end) rows gather sample 0 / row 0 and are zeroed afterwards
        const float* base_a = tm.src + (size_t)max(rn[i], 0) * tm.src_rows * tm.src_stride + f;
        const float* base_b = tm.src + (size_t)max(rn[i + 1], 0) * tm.src_rows * tm.src_stride + f;
        if (tm.op.idx == nullptr) {
          a = ldg4(base_a + (size_t)rr[i] * tm.src_stride);
          b = ldg4(base_b + (size_t)rr[i + 1] * tm.src_stride);
        } else {
          ell_gather4_pair(tm.op, rr[i], rr[i + 1], base_a, base_b, (size_t)tm.src_stride, a, b);
        }
        if (rn[i] < 0) a = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rn[i + 1] < 0) b = make_float4(0.f, 0.f, 0.f, 0.f);
        if (tm.stash != nullptr && do_stash) {    // keep the basis rows for the weight gradient (cape_term.stash)
          if (rn[i] >= 0) *reinterpret_cast<float4*>(tm.stash + (size_t)(row0 + rs + 32 * i) * tm.stash_stride + f) = a;
          if (rn[i + 1] >= 0)
            *reinterpret_cast<float4*>(tm.stash + (size_t)(row0 + rs + 32 * i + 32) * tm.stash_stride + f) = b;
        }
      }
      ra[i] = a; ra[i + 1] = b;
    }
    const bool has2 = DUAL && tm.w2T != nullptr;
#pragma unroll
    for (int i = 0; i < BN / 32; ++i) {
      const int c = col0 + rs + 32 * i;
      rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < p.ncols && f < tm.F) rb[i] = ldg4(tm.wT + (size_t)c * tm.wT_stride + f);
      if (DUAL) {
        rb2[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (has2 && c < p.ncols && f < tm.F) rb2[i] = ldg4(tm.w2T + (size_t)c * tm.w2T_stride + f);
      }
    }
  };
  auto store_chunk = [&](int stage) {
    char* a_hi = smem + (size_t)stage * Cfg::STAGE;
    char* a_lo = a_hi + A_TILE;
    char* b_hi = a_lo + A_TILE;
    char* b_lo = b_hi + Cfg::B_TILE;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = rs + 32 * i;
      split_store4(ra[i], a_hi, a_lo, (uint32_t)(row * 128 + ((l8 ^ (row & 7)) << 4)));
    }
#pragma unroll
    for (int i = 0; i < BN / 32; ++i) {
      const int cl = rs + 32 * i;
      const uint32_t off = (uint32_t)(cl * 128 + ((l8 ^ (cl & 7)) << 4));
      split_store4(rb[i], b_hi, b_lo, off);
      if (DUAL) split_store4(rb2[i], b_lo + Cfg::B_TILE, b_lo + 2 * Cfg::B_TILE, off);
    }
  };

  float acc0[NA], acc1[DUAL ? NA : 1], part0[NA], part1[DUAL ? NA : 1];
#pragma unroll
  for (int i = 0; i < NA; ++i) { acc0[i] = 0.f; if (DUAL) acc1[i] = 0.f; }

  // the reduction: 32-deep chunks over all terms
  int t = 0, f0 = 0;
  load_chunk(0, 0);
  store_chunk(0);
  fence_proxy_async();
  __syncthreads();
  for (int j = 0, stage = 0;; ++j, stage ^= 1) {
    const uint32_t a_hi = smem_u32(smem + (size_t)stage * Cfg::STAGE) + (uint32_t)(wgi * 64 * 128);
    const uint32_t a_lo = a_hi + A_TILE;
    const uint32_t b_hi = smem_u32(smem + (size_t)stage * Cfg::STAGE) + 2 * A_TILE;
    const uint32_t b_lo = b_hi + Cfg::B_TILE;
    wgmma_fence();
    fence_acc(part0);
    mma3_chunk<BN>(part0, a_hi, a_lo, b_hi, b_lo, 0);
    if constexpr (DUAL) {
      fence_acc(part1);
      mma3_chunk<BN>(part1, a_hi, a_lo, b_lo + Cfg::B_TILE, b_lo + 2 * Cfg::B_TILE, 0);
    }
    wgmma_commit();
    // next chunk: its loads fly while the MMAs run; the other stage was released at the end of the previous pass
    f0 += BK;
    if (f0 >= p.terms[t].F) { f0 = 0; ++t; }
    const bool more = t < p.nterms;
    if (more) {
      load_chunk(t, f0);
      store_chunk(stage ^ 1);
    }
    wgmma_wait_all();
    fence_acc(part0);
#pragma unroll
    for (int i = 0; i < NA; ++i) acc0[i] += part0[i];
    if constexpr (DUAL) {
      fence_acc(part1);
#pragma unroll
      for (int i = 0; i < NA; ++i) acc1[i] += part1[i];
    }
    if (!more) break;
    fence_proxy_async();            // generic-proxy smem writes -> visible to the tensor core's (async) proxy
    __syncthreads();                // both warpgroups done with this stage, the next one complete
  }
  __syncthreads();                  // qs complete (written before the main loop, read below)

  // =========================== epilogue: straight from the accumulator registers ===========================
  const bool linear = p.epilogue == CAPE_EPI_LINEAR;
  const bool use_aux = p.epilogue == CAPE_EPI_SLOPE || p.epilogue == CAPE_EPI_DUALMASK;
#pragma unroll
  for (int h = 0; h < 2; ++h) {                       // the thread's two rows
    const int lrow = wgi * 64 + frag_row(wt, 2 * h);
    const long long R = row0 + lrow;
    if (R >= p.total_rows) continue;
    const int n = (int)(R / p.rows_out), r = (int)(R % p.rows_out);
    const size_t orow = (size_t)R * p.ncols;
    float coef[MAX_SLOTS];
    for (int slot = 0; slot < p.nslots; ++slot) {
      const TermDev& tm = p.terms[p.slot_term[slot]];
      coef[slot] = tm.op.rowsum ? __ldg(tm.op.rowsum + r) : 1.f;
    }
    const float* bias_row = (linear && p.bias != nullptr) ? p.bias + (p.bias_per_row ? (size_t)r * p.ncols : 0) : nullptr;
#pragma unroll
    for (int g = 0; g < NA / 4; ++g) {
      const int i = 4 * g + 2 * h;
      const int c = col0 + frag_col(wt, i);
      if (c >= p.ncols) continue;
      float v0[2] = {acc0[i], acc0[i + 1]}, v1[2] = {0.f, 0.f};
      if (DUAL) { v1[0] = acc1[i]; v1[1] = acc1[i + 1]; }
      for (int slot = 0; slot < p.nslots; ++slot) {
        const float* q = qs + ((size_t)(n - n_first) * p.nslots + slot) * BN + (c - col0);
        if (p.slot_acc[slot] == 0) {
          v0[0] = fmaf(coef[slot], q[0], v0[0]); v0[1] = fmaf(coef[slot], q[1], v0[1]);
        } else if (DUAL) {
          v1[0] = fmaf(coef[slot], q[0], v1[0]); v1[1] = fmaf(coef[slot], q[1], v1[1]);
        }
      }
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
  }
}

template <int BN, bool DUAL>
int launch_conv(const ConvParams& p, cudaStream_t st) {
  using Cfg = ConvCfg<BN, DUAL>;
  int nqs = 0;
  if (p.nslots > 0) {
    const long long rlast_max = BM - 1;
    const int S = (int)(rlast_max / p.rows_out) + 2;
    nqs = S * p.nslots * BN;
  }
  const int smem = 1024 + Cfg::RING + nqs * 4;
  static bool configured = false;
  if (!configured) {
    CAPE_CHECK_CUDA(cudaFuncSetAttribute(conv_wg_kernel<BN, DUAL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         1024 + Cfg::RING + QS_MAX_FLOATS * 4));
    configured = true;
  }
  dim3 grid((unsigned)((p.total_rows + BM - 1) / BM), (unsigned)((p.ncols + BN - 1) / BN));
  conv_wg_kernel<BN, DUAL><<<grid, WG_THREADS, smem, st>>>(p, nqs);
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
  (void)t;
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
  if (kred < 64) return 0;                       // tiny reductions: the SIMT kernel is as good and simpler
  const int bn = pick_bn(p.ncols, dual);
  if (!qs_fits(p, bn)) return 0;
  if (dual) return bn == 32 ? launch_conv<32, true>(p, st) : launch_conv<64, true>(p, st);
  if (bn == 32) return launch_conv<32, false>(p, st);
  if (bn == 64) return launch_conv<64, false>(p, st);
  return launch_conv<128, false>(p, st);
}

// all-plain-operand calls: 1 = launched, 0 = not eligible (the caller falls through to the gather kernels)
int launch_gemm_tc(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st) {
  (void)t;
  if (!tensor_cores_enabled() || g_tuning[8] == 1) return 0;
  if (dual || p.epilogue == CAPE_EPI_AFFINE) return 0;
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
  if (bn == 32) return launch_conv<32, false>(p, st);
  if (bn == 64) return launch_conv<64, false>(p, st);
  return launch_conv<128, false>(p, st);
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
