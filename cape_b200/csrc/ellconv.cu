// Fused ELL-gather + contraction kernels (fp32 SIMT path).
//
// One kernel form serves the forward of chebyshev5 (+pool/unpool/bias/act/condition broadcast,
// reference lib/models.py:69-109,129-152,776-793,813-832) and its data gradient (same form with
// transposed operators/weights): each CTA owns a [128 rows x BN cols] output tile, builds the
// Chebyshev-basis tile A_t = op_t(src_t) chunk by chunk in shared memory from coalesced float4
// neighbour-row reads, and contracts it with the weight tile.  Nothing but the final activation
// is written to HBM: no transposes, no stacked basis, no materialised condition channels.
#include "common.cuh"
#include "ellconv_params.cuh"

namespace cape {

// ---- A-tile gather ------------------------------------------------------------------------------
__device__ __forceinline__ void gather_A(const TermDev& tm, int f0, const int* s_n, const int* s_r, int tid,
                                         float (&ra)[16]) {
  if (tm.vec) {
    const int l8 = tid & 7, rs = tid >> 3;
    const int f = f0 + l8 * 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = rs + 32 * i;
      const int n = s_n[row], r = s_r[row];
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n >= 0 && f < tm.F) {
        const float* base = tm.src + (size_t)n * tm.src_rows * tm.src_stride + f;
        if (tm.op.idx == nullptr) {
          v = ldg4(base + (size_t)r * tm.src_stride);
        } else {
          ell_gather4(tm.op, r, base, (size_t)tm.src_stride, v);
        }
      }
      ra[4 * i + 0] = v.x; ra[4 * i + 1] = v.y; ra[4 * i + 2] = v.z; ra[4 * i + 3] = v.w;
    }
  } else {
    const int lane = tid & 31, rs = tid >> 5;
    const int f = f0 + lane;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int row = rs + 8 * i;
      const int n = s_n[row], r = s_r[row];
      float v = 0.f;
      if (n >= 0 && f < tm.F) {
        const float* base = tm.src + (size_t)n * tm.src_rows * tm.src_stride + f;
        if (tm.op.idx == nullptr) v = __ldg(base + (size_t)r * tm.src_stride);
        else v = ell_gather1(tm.op, r, base, (size_t)tm.src_stride);
      }
      ra[i] = v;
    }
  }
}

__device__ __forceinline__ void store_A(int vec, int tid, const float (&ra)[16], float* As) {
  if (vec) {
    const int l8 = tid & 7, rs = tid >> 3;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      *reinterpret_cast<float4*>(&As[(rs + 32 * i) * AS_STRIDE + l8 * 4]) =
          make_float4(ra[4 * i], ra[4 * i + 1], ra[4 * i + 2], ra[4 * i + 3]);
  } else {
    const int lane = tid & 31, rs = tid >> 5;
#pragma unroll
    for (int i = 0; i < 16; ++i) As[(rs + 8 * i) * AS_STRIDE + lane] = ra[i];
  }
}

// ---- W-tile load ---------------------------------------------------------------------------------
template <int BN>
__device__ __forceinline__ void load_W(const float* w, int w_stride, int F, int f0, int col0, int ncols, int wvec,
                                       int tid, float (&rw)[BK * BN / NT]) {
  constexpr int WPT = BK * BN / NT;
  if (w == nullptr) {
#pragma unroll
    for (int i = 0; i < WPT; ++i) rw[i] = 0.f;
    return;
  }
  if (wvec) {
#pragma unroll
    for (int ps = 0; ps < WPT / 4; ++ps) {
      const int e4 = tid + NT * ps;
      const int kk = e4 / (BN / 4), c = (e4 % (BN / 4)) * 4;
      const int f = f0 + kk;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < F && col0 + c < ncols) v = ldg4(w + (size_t)f * w_stride + col0 + c);
      rw[4 * ps] = v.x; rw[4 * ps + 1] = v.y; rw[4 * ps + 2] = v.z; rw[4 * ps + 3] = v.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < WPT; ++i) {
      const int e = tid + NT * i;
      const int kk = e / BN, c = e % BN;
      const int f = f0 + kk;
      rw[i] = (f < F && col0 + c < ncols) ? __ldg(w + (size_t)f * w_stride + col0 + c) : 0.f;
    }
  }
}

template <int BN>
__device__ __forceinline__ void store_W(int wvec, int tid, const float (&rw)[BK * BN / NT], float* Ws) {
  constexpr int WPT = BK * BN / NT;
  if (wvec) {
#pragma unroll
    for (int ps = 0; ps < WPT / 4; ++ps) {
      const int e4 = tid + NT * ps;
      const int kk = e4 / (BN / 4), c = (e4 % (BN / 4)) * 4;
      *reinterpret_cast<float4*>(&Ws[kk * BN + c]) = make_float4(rw[4 * ps], rw[4 * ps + 1], rw[4 * ps + 2], rw[4 * ps + 3]);
    }
  } else {
#pragma unroll
    for (int i = 0; i < WPT; ++i) {
      const int e = tid + NT * i;
      Ws[(e / BN) * BN + (e % BN)] = rw[i];
    }
  }
}

template <int RPT, int TY, int BN>
__device__ __forceinline__ void mac_tile(const float* As, const float* Ws, int tx, int ty, float (&acc)[RPT][4]) {
#pragma unroll
  for (int kk = 0; kk < BK; kk += 4) {
    float4 b[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) b[u] = *reinterpret_cast<const float4*>(&Ws[(kk + u) * BN + tx * 4]);
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
      const float4 a = *reinterpret_cast<const float4*>(&As[(ty + TY * i) * AS_STRIDE + kk]);
      acc[i][0] = fmaf(a.x, b[0].x, acc[i][0]); acc[i][1] = fmaf(a.x, b[0].y, acc[i][1]);
      acc[i][2] = fmaf(a.x, b[0].z, acc[i][2]); acc[i][3] = fmaf(a.x, b[0].w, acc[i][3]);
      acc[i][0] = fmaf(a.y, b[1].x, acc[i][0]); acc[i][1] = fmaf(a.y, b[1].y, acc[i][1]);
      acc[i][2] = fmaf(a.y, b[1].z, acc[i][2]); acc[i][3] = fmaf(a.y, b[1].w, acc[i][3]);
      acc[i][0] = fmaf(a.z, b[2].x, acc[i][0]); acc[i][1] = fmaf(a.z, b[2].y, acc[i][1]);
      acc[i][2] = fmaf(a.z, b[2].z, acc[i][2]); acc[i][3] = fmaf(a.z, b[2].w, acc[i][3]);
      acc[i][0] = fmaf(a.w, b[3].x, acc[i][0]); acc[i][1] = fmaf(a.w, b[3].y, acc[i][1]);
      acc[i][2] = fmaf(a.w, b[3].z, acc[i][2]); acc[i][3] = fmaf(a.w, b[3].w, acc[i][3]);
    }
  }
}

// PASS: the call has pass-through terms (see conv_wg_kernel)
template <int BN, bool DUAL, bool PASS>
__global__ void __launch_bounds__(NT, DUAL ? 1 : 2) ellconv_kernel(const __grid_constant__ ConvParams p) {
  constexpr int TX = BN / 4, TY = NT / TX, RPT = BM / TY;
  constexpr int WPT = BK * BN / NT;
  __shared__ __align__(16) float As[BM * AS_STRIDE];
  __shared__ __align__(16) float Ws[BK * BN];
  __shared__ __align__(16) float Ws2[DUAL ? BK * BN : 4];
  __shared__ int s_n[BM], s_r[BM];

  const int tid = threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const long long row0 = (long long)blockIdx.x * BM;
  const int col0 = blockIdx.y * BN;

  if (tid < BM) {
    const long long R = row0 + tid;
    if (R < p.total_rows) {
      s_n[tid] = (int)(R / p.rows_out);
      s_r[tid] = (int)(R % p.rows_out);
    } else {
      s_n[tid] = -1;
      s_r[tid] = 0;
    }
  }
  __syncthreads();

  float acc0[RPT][4];
  float acc1[RPT][4];
#pragma unroll
  for (int i = 0; i < RPT; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc0[i][j] = 0.f;
#pragma unroll
  for (int i = 0; i < RPT; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc1[i][j] = 0.f;

  float ra[16];
  float rw[WPT];
  float rw2[WPT];

  int t = 0, f0 = 0;            // chunk currently held in registers
  gather_A(p.terms[0], 0, s_n, s_r, tid, ra);
  load_W<BN>(p.terms[0].w, p.terms[0].w_stride, p.terms[0].F, 0, col0, p.ncols, p.wvec, tid, rw);
  if (DUAL) load_W<BN>(p.terms[0].w2, p.terms[0].w2_stride, p.terms[0].F, 0, col0, p.ncols, p.wvec, tid, rw2);

  while (t < p.nterms) {
    const bool has2 = DUAL && (p.terms[t].w2 != nullptr);
    store_A(p.terms[t].vec, tid, ra, As);
    store_W<BN>(p.wvec, tid, rw, Ws);
    if (has2) store_W<BN>(p.wvec, tid, rw2, Ws2);
    __syncthreads();
    // advance to the next chunk and prefetch it while computing the current one
    int nt = t, nf0 = f0 + BK;
    if (nf0 >= p.terms[t].F) { nt = t + 1; nf0 = 0; }
    if (nt < p.nterms) {
      gather_A(p.terms[nt], nf0, s_n, s_r, tid, ra);
      load_W<BN>(p.terms[nt].w, p.terms[nt].w_stride, p.terms[nt].F, nf0, col0, p.ncols, p.wvec, tid, rw);
      if (DUAL) load_W<BN>(p.terms[nt].w2, p.terms[nt].w2_stride, p.terms[nt].F, nf0, col0, p.ncols, p.wvec, tid, rw2);
    }
    mac_tile<RPT, TY, BN>(As, Ws, tx, ty, acc0);
    if (DUAL) {
      if (has2) mac_tile<RPT, TY, BN>(As, Ws2, tx, ty, acc1);
    }
    __syncthreads();
    t = nt; f0 = nf0;
  }

  // ---- condition broadcast, staged in As ---------------------------------------------------------
  float* qs = As;
  const int n_first = s_n[0];
  if (p.nslots > 0) {
    int n_last = n_first;
    for (int i = BM - 1; i > 0; --i)
      if (s_n[i] >= 0) { n_last = s_n[i]; break; }
    stage_cond<16>(p, qs, n_first, n_last - n_first + 1, col0, BN, p.ncols, tid, NT);
    __syncthreads();
  }

  // ---- epilogue (the tanh ones compiled out with two accumulators: refused by cape_cheb_fwd) ----------
  const EpiParams& e = p.epi;
#pragma unroll
  for (int i = 0; i < RPT; ++i) {
    const int row = ty + TY * i;
    const int n = s_n[row];
    if (n < 0) continue;
    const int r = s_r[row];
    float v0[4], v1[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { v0[j] = acc0[i][j]; v1[j] = DUAL ? acc1[i][j] : 0.f; }
    for (int slot = 0; slot < p.nslots; ++slot) {
      const float coef = cond_coef(p.terms[p.slot_term[slot]].op, r);
      const float* q = cond_vec(qs, n - n_first, slot, p.nslots, BN) + tx * 4;
      if (p.slot_acc[slot] == 0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) v0[j] = fmaf(coef, q[j], v0[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) v1[j] = fmaf(coef, q[j], v1[j]);
      }
    }
    const int c0 = col0 + tx * 4;
    if constexpr (PASS) {
      for (int q = p.nterms; q < p.nterms + p.npass; ++q) {   // pass-through terms (F == ncols)
        const TermDev& tm = p.terms[q];
        const float* base = tm.src + (size_t)n * tm.src_rows * tm.src_stride;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (c0 + j < p.ncols) v0[j] += pass_row(tm.op, r, base + c0 + j, (size_t)tm.src_stride);
      }
    }
    const size_t obase = ((size_t)(row0 + row)) * p.ncols + c0;
    float b[4] = {0.f, 0.f, 0.f, 0.f}, ax[4] = {0.f, 0.f, 0.f, 0.f}, o1[4], o2[4];
    if (e.epilogue == CAPE_EPI_LINEAR && e.bias != nullptr) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (c0 + j < p.ncols) b[j] = __ldg(e.bias + (e.bias_per_row ? (size_t)r * p.ncols : 0) + c0 + j);
    } else if (epi_reads_aux(e.epilogue)) {
      if (p.ovec && c0 < p.ncols) {
        const float4 a4 = ldg4(e.aux + obase);
        ax[0] = a4.x; ax[1] = a4.y; ax[2] = a4.z; ax[3] = a4.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) ax[j] = (c0 + j < p.ncols) ? __ldg(e.aux + obase + j) : 0.f;
      }
    }
    const bool write2 = apply_epilogue<!DUAL>(e, v0, v1, b, ax, o1, o2);
    if (p.ovec) {
      if (c0 < p.ncols) {
        *reinterpret_cast<float4*>(e.out + obase) = make_float4(o1[0], o1[1], o1[2], o1[3]);
        if (write2) *reinterpret_cast<float4*>(e.out2 + obase) = make_float4(o2[0], o2[1], o2[2], o2[3]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (c0 + j < p.ncols) {
          e.out[obase + j] = o1[j];
          if (write2) e.out2[obase + j] = o2[j];
        }
    }
  }
}

// ---- weight-gradient kernel -----------------------------------------------------------------------
constexpr int DW_BF = 64, DW_BC = 64, DW_BR = 32, DW_STRIDE = 68;

struct DwParams {
  int N, rows_out, ncols;
  long long total_rows;
  long long rows_per_split;
  const float* src;
  OpView op;
  int F, src_rows, src_stride;
  const float* g;
  float* out;          // either dw (nsplit == 1) or workspace [nsplit, F, ncols]
  long long out_rs;    // row stride of out
  int nsplit;
  int accumulate;
  int vec, gvec;
};

__device__ __forceinline__ void dw_gather(const DwParams& p, long long rbase, long long rend, int ftile, int tid,
                                          float (&ra)[8]) {
  if (p.vec) {
    const int l16 = tid & 15, rs = tid >> 4;
    const int f = ftile + l16 * 4;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const long long R = rbase + rs + 16 * i;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (R < rend && f < p.F) {
        const int n = (int)(R / p.rows_out), r = (int)(R % p.rows_out);
        const float* base = p.src + (size_t)n * p.src_rows * p.src_stride + f;
        if (p.op.idx == nullptr) {
          v = ldg4(base + (size_t)r * p.src_stride);
        } else {
          ell_gather4(p.op, r, base, (size_t)p.src_stride, v);
        }
      }
      ra[4 * i] = v.x; ra[4 * i + 1] = v.y; ra[4 * i + 2] = v.z; ra[4 * i + 3] = v.w;
    }
  } else {
    const int lane = tid & 63, rs = tid >> 6;
    const int f = ftile + lane;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const long long R = rbase + rs + 4 * i;
      float v = 0.f;
      if (R < rend && f < p.F) {
        const int n = (int)(R / p.rows_out), r = (int)(R % p.rows_out);
        const float* base = p.src + (size_t)n * p.src_rows * p.src_stride + f;
        if (p.op.idx == nullptr) v = __ldg(base + (size_t)r * p.src_stride);
        else v = ell_gather1(p.op, r, base, (size_t)p.src_stride);
      }
      ra[i] = v;
    }
  }
}

__device__ __forceinline__ void dw_load_g(const DwParams& p, long long rbase, long long rend, int ctile, int tid,
                                          float (&rg)[8]) {
  if (p.gvec) {
    const int l16 = tid & 15, rs = tid >> 4;
    const int c = ctile + l16 * 4;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const long long R = rbase + rs + 16 * i;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (R < rend && c < p.ncols) v = ldg4(p.g + (size_t)R * p.ncols + c);
      rg[4 * i] = v.x; rg[4 * i + 1] = v.y; rg[4 * i + 2] = v.z; rg[4 * i + 3] = v.w;
    }
  } else {
    const int lane = tid & 63, rs = tid >> 6;
    const int c = ctile + lane;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const long long R = rbase + rs + 4 * i;
      rg[i] = (R < rend && c < p.ncols) ? __ldg(p.g + (size_t)R * p.ncols + c) : 0.f;
    }
  }
}

__device__ __forceinline__ void dw_store(int vec, int tid, const float (&r)[8], float* S) {
  if (vec) {
    const int l16 = tid & 15, rs = tid >> 4;
#pragma unroll
    for (int i = 0; i < 2; ++i)
      *reinterpret_cast<float4*>(&S[(rs + 16 * i) * DW_STRIDE + l16 * 4]) =
          make_float4(r[4 * i], r[4 * i + 1], r[4 * i + 2], r[4 * i + 3]);
  } else {
    const int lane = tid & 63, rs = tid >> 6;
#pragma unroll
    for (int i = 0; i < 8; ++i) S[(rs + 4 * i) * DW_STRIDE + lane] = r[i];
  }
}

__global__ void __launch_bounds__(NT, 2) ellconv_dw_kernel(const __grid_constant__ DwParams p) {
  __shared__ __align__(16) float As[DW_BR * DW_STRIDE];
  __shared__ __align__(16) float Gs[DW_BR * DW_STRIDE];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int ftile = blockIdx.x * DW_BF, ctile = blockIdx.y * DW_BC;
  const long long rbeg = (long long)blockIdx.z * p.rows_per_split;
  const long long rend = min(p.total_rows, rbeg + p.rows_per_split);

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  float ra[8], rg[8];
  if (rbeg < rend) {
    dw_gather(p, rbeg, rend, ftile, tid, ra);
    dw_load_g(p, rbeg, rend, ctile, tid, rg);
  }
  for (long long rb = rbeg; rb < rend; rb += DW_BR) {
    dw_store(p.vec, tid, ra, As);
    dw_store(p.gvec, tid, rg, Gs);
    __syncthreads();
    if (rb + DW_BR < rend) {
      dw_gather(p, rb + DW_BR, rend, ftile, tid, ra);
      dw_load_g(p, rb + DW_BR, rend, ctile, tid, rg);
    }
#pragma unroll 8
    for (int rr = 0; rr < DW_BR; ++rr) {
      const float4 a = *reinterpret_cast<const float4*>(&As[rr * DW_STRIDE + ty * 4]);
      const float4 g = *reinterpret_cast<const float4*>(&Gs[rr * DW_STRIDE + tx * 4]);
      acc[0][0] = fmaf(a.x, g.x, acc[0][0]); acc[0][1] = fmaf(a.x, g.y, acc[0][1]);
      acc[0][2] = fmaf(a.x, g.z, acc[0][2]); acc[0][3] = fmaf(a.x, g.w, acc[0][3]);
      acc[1][0] = fmaf(a.y, g.x, acc[1][0]); acc[1][1] = fmaf(a.y, g.y, acc[1][1]);
      acc[1][2] = fmaf(a.y, g.z, acc[1][2]); acc[1][3] = fmaf(a.y, g.w, acc[1][3]);
      acc[2][0] = fmaf(a.z, g.x, acc[2][0]); acc[2][1] = fmaf(a.z, g.y, acc[2][1]);
      acc[2][2] = fmaf(a.z, g.z, acc[2][2]); acc[2][3] = fmaf(a.z, g.w, acc[2][3]);
      acc[3][0] = fmaf(a.w, g.x, acc[3][0]); acc[3][1] = fmaf(a.w, g.y, acc[3][1]);
      acc[3][2] = fmaf(a.w, g.z, acc[3][2]); acc[3][3] = fmaf(a.w, g.w, acc[3][3]);
    }
    __syncthreads();
  }

  float* out = p.out;
  if (p.nsplit > 1) out += (size_t)blockIdx.z * p.F * p.out_rs;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int f = ftile + ty * 4 + i;
    if (f >= p.F) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = ctile + tx * 4 + j;
      if (c >= p.ncols) continue;
      float* o = out + (size_t)f * p.out_rs + c;
      if (p.nsplit == 1 && p.accumulate) *o += acc[i][j];
      else *o = acc[i][j];
    }
  }
}

// rows q of the partial blocks go to  dw + (q % Fper) * dw_stride + (q / Fper) * term_stride  (several terms at once)
__global__ void __launch_bounds__(1024) reduce_splits_kernel(const float* __restrict__ ws, int nsplit, int F, int ncols,
                                                             float* __restrict__ dw, long long dw_stride,
                                                             int accumulate, int Fper, long long term_stride,
                                                             long long col_stride) {
  // 32 consecutive elements x 32 split lanes per CTA (a 64 x 64 gradient with ~300 partials: 128 CTAs, nine loads per
  // thread); fixed summation order (deterministic)
  __shared__ float red[32][33];
  const long long total = (long long)F * ncols;
  const int el = threadIdx.x & 31, zl = threadIdx.x >> 5;
  for (long long e0 = (long long)blockIdx.x * 32; e0 < total; e0 += (long long)gridDim.x * 32) {
    const long long e = e0 + el;
    float s = 0.f;
    if (e < total) {
#pragma unroll 4
      for (int z = zl; z < nsplit; z += 32) s += ws[(size_t)z * total + e];
    }
    red[zl][el] = s;
    __syncthreads();
    if (zl == 0 && e < total) {
      s = 0.f;
#pragma unroll
      for (int k = 0; k < 32; ++k) s += red[k][el];
      const int q = (int)(e / ncols), c = (int)(e % ncols);
      float* o = dw + (size_t)(q % Fper) * dw_stride + (size_t)(q / Fper) * term_stride + (size_t)c * col_stride;
      *o = accumulate ? (*o + s) : s;
    }
    __syncthreads();
  }
}

// ---- per-sample weighted column sums ------------------------------------------------------------------
constexpr int CS_MAXOPS = 4;
struct ColsumParams {
  const float* g;
  int N, rows, ncols, nops, rows_per_block, vec, gs;   // gs: floats between consecutive rows of g
  const float* coef[CS_MAXOPS];   // nullptr = ones
  float* out;
};

__global__ void __launch_bounds__(256) colsum_kernel(const __grid_constant__ ColsumParams p) {
  // grid: (row blocks, N).  Threads = (ncols/4 float4 column lanes) x (row lanes); every row is read as one
  // contiguous ncols*4-byte segment.  Scalar fallback when ncols % 4 != 0.
  __shared__ float red[CS_MAXOPS][256 * 4 / 32][33];   // [op][row lane (<=32)][col4 lane*4 .. ] reused below
  const int n = blockIdx.y;
  const int r0 = blockIdx.x * p.rows_per_block;
  const int r1 = min(p.rows, r0 + p.rows_per_block);
  const float* gp = p.g + (size_t)n * p.rows * p.gs;
  if (p.vec) {
    const int cl = p.ncols >> 2;                       // float4 lanes per row (<= 128)
    const int rl = 256 / cl;                           // row lanes
    const int c4 = threadIdx.x % cl, ry = threadIdx.x / cl;
    float4 s[CS_MAXOPS];
#pragma unroll
    for (int j = 0; j < CS_MAXOPS; ++j) s[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ry < rl) {
      int r = r0 + ry;
      // four rows per trip: their loads are independent, so they are all in flight before the first FMA needs one
      for (; r + 3 * rl < r1; r += 4 * rl) {
        const float* g0 = gp + (size_t)r * p.gs + c4 * 4;
        const size_t step = (size_t)rl * p.gs;
        const float4 v0 = ldg4(g0), v1 = ldg4(g0 + step), v2 = ldg4(g0 + 2 * step), v3 = ldg4(g0 + 3 * step);
#pragma unroll
        for (int j = 0; j < CS_MAXOPS; ++j)
          if (j < p.nops) {
            const float* cf = p.coef[j];
            const float k0 = cf ? __ldg(cf + r) : 1.f, k1 = cf ? __ldg(cf + r + rl) : 1.f;
            const float k2 = cf ? __ldg(cf + r + 2 * rl) : 1.f, k3 = cf ? __ldg(cf + r + 3 * rl) : 1.f;
            fma4(s[j], k0, v0); fma4(s[j], k1, v1); fma4(s[j], k2, v2); fma4(s[j], k3, v3);
          }
      }
      for (; r < r1; r += rl) {
        const float4 gv = ldg4(gp + (size_t)r * p.gs + c4 * 4);
#pragma unroll
        for (int j = 0; j < CS_MAXOPS; ++j)
          if (j < p.nops) fma4(s[j], p.coef[j] ? __ldg(p.coef[j] + r) : 1.f, gv);
      }
    }
    // reduce over row lanes through shared memory (fixed order), then one atomic per (op, column)
    float* sm = &red[0][0][0];                         // 4 * 32 * 33 floats = 4224 >= nops * 256 * 4 when rl*cl = 256
    for (int j = 0; j < p.nops; ++j) {
      __syncthreads();
      if (ry < rl) *reinterpret_cast<float4*>(sm + ((size_t)ry * cl + c4) * 4) = s[j];
      __syncthreads();
      for (int c = threadIdx.x; c < p.ncols; c += 256) {
        float tot = 0.f;
        for (int k = 0; k < rl; ++k) tot += sm[((size_t)k * cl + (c >> 2)) * 4 + (c & 3)];
        atomicAdd(p.out + ((size_t)n * p.nops + j) * p.ncols + c, tot);
      }
    }
  } else {
    const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
    for (int c0 = 0; c0 < p.ncols; c0 += 32) {
      const int c = c0 + cx;
      float s[CS_MAXOPS] = {0.f, 0.f, 0.f, 0.f};
      if (c < p.ncols)
        for (int r = r0 + ry; r < r1; r += 8) {
          const float gv = __ldg(gp + (size_t)r * p.gs + c);
#pragma unroll
          for (int j = 0; j < CS_MAXOPS; ++j)
            if (j < p.nops) s[j] = fmaf(p.coef[j] ? __ldg(p.coef[j] + r) : 1.f, gv, s[j]);
        }
      __syncthreads();
#pragma unroll
      for (int j = 0; j < CS_MAXOPS; ++j) red[j][ry][cx] = s[j];
      __syncthreads();
      if (ry == 0 && c < p.ncols)
        for (int j = 0; j < p.nops; ++j) {
          float tot = 0.f;
#pragma unroll
          for (int k = 0; k < 8; ++k) tot += red[j][k][cx];
          atomicAdd(p.out + ((size_t)n * p.nops + j) * p.ncols + c, tot);
        }
    }
  }
}

// ---- standalone resampling (poolwT, lib/models.py:129-152): y[n, r, :F] = sum_j w[r, j] * x[n, idx[r, j], :F] -------
// x rows are xs floats apart, y rows ys floats apart (so the result can land inside a wider concat buffer);
// op.idx == nullptr copies rows (identity).  Optionally the condition channels of the concat are written too:
// y[n, r, F + c] = rowsum(op)[r] * cond[n, c]   (fit_cond_dim + concat + unpool, lib/models.py:606-609,750).
__global__ void __launch_bounds__(256) resample_kernel(OpView op, const float* __restrict__ x, int xs,
                                                       float* __restrict__ y, int ys, long long total_rows,
                                                       int rows_out, int rows_in, int F, int vec,
                                                       const float* __restrict__ cond, int C) {
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= total_rows) return;
  const int n = (int)(warp / rows_out), r = (int)(warp % rows_out);
  const float* base = x + (size_t)n * rows_in * xs;
  float* out = y + (size_t)warp * ys;
  if (vec) {
    for (int f = lane * 4; f < F; f += 128) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (op.idx == nullptr) v = ldg4(base + (size_t)r * xs + f);
      else ell_gather4(op, r, base + f, (size_t)xs, v);
      *reinterpret_cast<float4*>(out + f) = v;
    }
  } else {
    for (int f = lane; f < F; f += 32) {
      out[f] = op.idx == nullptr ? __ldg(base + (size_t)r * xs + f) : ell_gather1(op, r, base + f, (size_t)xs);
    }
  }
  if (cond != nullptr) {
    const float coef = cond_coef(op, r);
    for (int c = lane; c < C; c += 32) out[F + c] = coef * __ldg(cond + (size_t)n * C + c);
  }
}

}  // namespace cape

using namespace cape;

extern "C" int cape_resample(cape_topology* t, int op, const float* x, int x_stride, float* y, int y_stride, int N,
                             int rows_out, int rows_in, int F, const float* cond, int C, void* stream) {
  CAPE_REQUIRE(t && x && y && N > 0 && F > 0, "bad arguments");
  CAPE_REQUIRE(x_stride >= F && y_stride >= F + (cond ? C : 0), "bad strides");
  OpView v;
  if (get_op(t, op, rows_out, rows_in, &v) != 0) return -1;
  const long long total = (long long)N * rows_out;
  const int vec = (F % 4 == 0) && (x_stride % 4 == 0) && (y_stride % 4 == 0) && aligned16(x) && aligned16(y);
  const long long blocks = (total * 32 + 255) / 256;
  resample_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(v, x, x_stride, y, y_stride, total, rows_out,
                                                                      rows_in, F, vec, cond, C);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_cheb_fwd(cape_topology* t, const cape_conv_args* a, void* stream) {
  CAPE_REQUIRE(t && a, "null handle/args");
  CAPE_REQUIRE(a->N > 0 && a->rows_out > 0 && a->ncols > 0, "empty problem");
  CAPE_REQUIRE(a->nterms >= 1 && a->nterms <= CAPE_MAX_TERMS, "nterms out of range");
  CAPE_REQUIRE(a->out != nullptr, "out is null");
  ConvParams p{};
  p.N = a->N; p.rows_out = a->rows_out; p.ncols = a->ncols; p.nterms = a->nterms;
  p.total_rows = (long long)a->N * a->rows_out;
  bool dual = false, any_stash = false;
  bool wvec = (a->ncols % 4 == 0);
  p.nslots = 0;
  // contracted terms first, in call order; pass-through terms (no weights at all) after them
  int npass = 0;
  for (int i = 0; i < a->nterms; ++i) {
    const cape_term& s = a->terms[i];
    if (s.w || s.w2 || s.wT || s.w2T) continue;
    CAPE_REQUIRE(!a->plain_only, "a pass-through term (no w, w2, wT or w2T) cannot be part of a plain_only call");
    CAPE_REQUIRE(s.src && s.F == a->ncols, "a pass-through term needs src and F == ncols");
    CAPE_REQUIRE(!s.wc && !s.wc2 && !s.stash, "a pass-through term takes no wc, wc2 or stash");
    CAPE_REQUIRE(s.src_stride >= s.F, "bad strides");
    ++npass;
  }
  CAPE_REQUIRE(npass < a->nterms, "a call needs at least one contracted term");
  p.nterms = a->nterms - npass;
  p.npass = npass;
  for (int i = 0, ic = 0, ip = p.nterms; i < a->nterms; ++i) {
    const cape_term& s = a->terms[i];
    if (!(s.w || s.w2 || s.wT || s.w2T)) {
      TermDev& d = p.terms[ip++];
      if (get_op(t, s.op, a->rows_out, s.src_rows, &d.op) != 0) return -1;
      d.src = s.src; d.F = s.F; d.src_rows = s.src_rows; d.src_stride = s.src_stride;
      d.vec = (s.F % 4 == 0) && (s.src_stride % 4 == 0) && aligned16(s.src);
      continue;
    }
    CAPE_REQUIRE(s.src && (s.w || a->plain_only) && s.F > 0, "term needs src, w and F > 0");
    CAPE_REQUIRE(s.src_stride >= s.F && (s.w_stride >= a->ncols || a->plain_only), "bad strides");
    const int ti = ic++;
    TermDev& d = p.terms[ti];
    if (get_op(t, s.op, a->rows_out, s.src_rows, &d.op) != 0) return -1;
    d.src = s.src; d.F = s.F; d.src_rows = s.src_rows; d.src_stride = s.src_stride; d.w_stride = s.w_stride; d.w2_stride = s.w2_stride;
    d.w = s.w; d.w2 = s.w2;
    d.wT = s.wT; d.w2T = s.w2T; d.wT_stride = s.wT_stride; d.w2T_stride = s.w2T_stride;
    d.vec = (s.F % 4 == 0) && (s.src_stride % 4 == 0) && aligned16(s.src);
    d.stash = s.stash; d.stash_stride = s.stash_stride;
    if (s.stash) {
      CAPE_REQUIRE(s.F % 4 == 0 && s.stash_stride >= s.F && s.stash_stride % 4 == 0 && aligned16(s.stash),
                   "stash needs F % 4 == 0, stash_stride % 4 == 0 and 16-byte alignment");
      any_stash = true;
    }
    wvec = wvec && (s.w_stride % 4 == 0) && aligned16(s.w) && (!s.w2 || aligned16(s.w2));
    if (s.w2) {
      dual = true;
      CAPE_REQUIRE(s.w2_stride >= a->ncols, "bad w2_stride");
      wvec = wvec && (s.w2_stride % 4 == 0);
    }
    if (s.wc) {
      CAPE_REQUIRE(a->cond && a->C > 0, "condition weights without cond");
      p.slot_term[p.nslots] = ti; p.slot_acc[p.nslots] = 0;
      p.slot_w[p.nslots] = s.wc; p.slot_ws[p.nslots] = s.w_stride; ++p.nslots;
    }
    if (s.wc2) {
      CAPE_REQUIRE(a->cond && a->C > 0 && s.w2, "wc2 needs cond and w2");
      p.slot_term[p.nslots] = ti; p.slot_acc[p.nslots] = 1;
      p.slot_w[p.nslots] = s.wc2; p.slot_ws[p.nslots] = s.w2_stride; ++p.nslots;
    }
  }
  p.cond = a->cond; p.C = a->C;
  if (fill_epilogue(a, dual, &p.epi) != 0) return -1;
  p.wvec = wvec ? 1 : 0;
  p.ovec = (a->ncols % 4 == 0) && aligned16(a->out) && (!a->out2 || aligned16(a->out2)) && (!a->aux || aligned16(a->aux));
  const int BNsel = a->ncols <= 32 ? 32 : 64;
  CAPE_REQUIRE(max_tile_samples(BM, a->rows_out) * p.nslots * BNsel <= BM * AS_STRIDE,
               "rows_out too small for the condition staging buffer");
  cudaStream_t st = (cudaStream_t)stream;
  if (a->plain_only) {
    const int rc = launch_gemm_tc(t, p, dual, st);
    if (rc != 0) return rc < 0 ? rc : 0;
    CAPE_REQUIRE(false, "plain_only call not eligible for the tensor-core contraction (needs the tensor-core path, all "
                        "terms identity with wT, ncols % 16 == 0, 16-byte aligned operands)");
  }
  {
    int rc = launch_thin_fwd(t, p, dual, st);             // <= 4 input channels: streaming kernel
    if (rc != 0) return rc < 0 ? rc : 0;
    rc = launch_thinout_fwd(t, p, dual, st);              // <= 4 output columns: contract first, then gather
    if (rc != 0) return rc < 0 ? rc : 0;
    rc = launch_gemm_tc(t, p, dual, st);                  // plain operands only: wgmma contraction
    if (rc != 0) return rc < 0 ? rc : 0;
    rc = launch_ellconv_tc(t, p, dual, st);               // wgmma path when eligible (writes the stashes itself)
    if (rc != 0) return rc < 0 ? rc : 0;
  }
  // the fp32-pipe kernel with two accumulators (the affine block's forward) has no tanh epilogues: they would cost it
  // registers it spills already
  CAPE_REQUIRE(!dual || !needs_tanh(p.epi),
               "tanh / TANHGRAD epilogues with a w2 term need the tensor-core kernel (ncols % 32 == 0, wT / w2T given)");
  if (any_stash) {                                        // fp32-pipe path: the basis copies come from the resample kernel
    for (int i = 0; i < p.nterms; ++i) {
      const TermDev& d = p.terms[i];
      if (!d.stash) continue;
      const long long blocks = (p.total_rows * 32 + 255) / 256;
      const int vec = d.vec && (d.stash_stride % 4 == 0);
      resample_kernel<<<(unsigned)blocks, 256, 0, st>>>(d.op, d.src, d.src_stride, d.stash, d.stash_stride, p.total_rows,
                                                        a->rows_out, d.src_rows, d.F, vec, nullptr, 0);
      CAPE_CHECK_CUDA(cudaGetLastError());
      cape::count_launches(1);
    }
  }
  dim3 grid((unsigned)((p.total_rows + BM - 1) / BM), (unsigned)((a->ncols + BNsel - 1) / BNsel));
  if (p.npass > 0) {
    if (dual) {
      if (BNsel == 32) ellconv_kernel<32, true, true><<<grid, NT, 0, st>>>(p);
      else ellconv_kernel<64, true, true><<<grid, NT, 0, st>>>(p);
    } else {
      if (BNsel == 32) ellconv_kernel<32, false, true><<<grid, NT, 0, st>>>(p);
      else ellconv_kernel<64, false, true><<<grid, NT, 0, st>>>(p);
    }
  } else if (dual) {
    if (BNsel == 32) ellconv_kernel<32, true, false><<<grid, NT, 0, st>>>(p);
    else ellconv_kernel<64, true, false><<<grid, NT, 0, st>>>(p);
  } else {
    if (BNsel == 32) ellconv_kernel<32, false, false><<<grid, NT, 0, st>>>(p);
    else ellconv_kernel<64, false, false><<<grid, NT, 0, st>>>(p);
  }
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

static int dw_single(cape_topology* t, const cape_dw_args* a, void* stream);

// sums the nsplit partial blocks [nsplit, F, ncols] of the workspace into dw (reduce_splits_kernel)
static int reduce_splits(const cape_topology* t, int nsplit, int F, int ncols, float* dw, long long dw_stride,
                         int accumulate, int Fper, long long term_stride, long long col_stride, cudaStream_t st) {
  const long long total = (long long)F * ncols;
  long long blocks = (total + 31) / 32;
  if (blocks > 8LL * t->sm_count) blocks = 8LL * t->sm_count;
  reduce_splits_kernel<<<(unsigned)blocks, 1024, 0, st>>>((const float*)t->workspace, nsplit, F, ncols, dw, dw_stride,
                                                          accumulate, Fper, term_stride, col_stride);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_cheb_dw(cape_topology* t, const cape_dw_args* a, void* stream) {
  CAPE_REQUIRE(t && a, "null handle/args");
  CAPE_REQUIRE(a->N > 0 && a->rows_out > 0 && a->ncols > 0 && a->F > 0, "empty problem");
  CAPE_REQUIRE(a->src && a->g && a->dw, "null pointer");
  CAPE_REQUIRE(a->src_stride >= a->F && (a->dw_stride >= a->ncols || a->dw_col_stride > 1), "bad strides");
  if (a->nops <= 0) {
    CAPE_REQUIRE(a->dw_col_stride <= 1, "dw_col_stride needs the multi-term form (nops > 0)");
    return dw_single(t, a, stream);
  }
  CAPE_REQUIRE(a->nops <= CAPE_MAX_TERMS, "nops out of range");
  // several terms of one layer: one pass over g when the input is thin, else term by term
  OpView ops[CAPE_MAX_TERMS];
  for (int j = 0; j < a->nops; ++j)
    if (get_op(t, a->ops[j], a->rows_out, a->src_rows, &ops[j]) != 0) return -1;
  int ns = 1;
  int rc = launch_thin_dw(t, a, ops, a->nops, &ns, (cudaStream_t)stream);
  if (rc < 0) return rc;
  if (rc == 1)
    return reduce_splits(t, ns, a->nops * a->F, a->ncols, a->dw, a->dw_stride, a->accumulate, a->F, a->dw_term_stride,
                         a->dw_col_stride > 0 ? a->dw_col_stride : 1, (cudaStream_t)stream);
  CAPE_REQUIRE(a->dw_col_stride <= 1, "dw_col_stride is only implemented for thin inputs (F <= 4, ncols 32..256)");
  for (int j = 0; j < a->nops; ++j) {
    cape_dw_args b = *a;
    b.nops = 0; b.op = a->ops[j]; b.dw = a->dw + (size_t)j * a->dw_term_stride;
    rc = dw_single(t, &b, stream);
    if (rc != 0) return rc;
  }
  return 0;
}

static int dw_single(cape_topology* t, const cape_dw_args* a, void* stream) {
  DwParams p{};
  if (get_op(t, a->op, a->rows_out, a->src_rows, &p.op) != 0) return -1;
  {
    int ns = 1;
    bool always_reduce = false;
    int rc = launch_thin_dw(t, a, &p.op, 1, &ns, (cudaStream_t)stream);           // <= 4 input channels
    if (rc < 0) return rc;
    if (rc == 1) always_reduce = true;                                            // partials always in the workspace
    else rc = launch_ellconv_dw_tc(t, a, p.op, &ns, (cudaStream_t)stream);        // tensor cores (wgmma)
    if (rc < 0) return rc;
    if (rc == 1) {
      if (ns > 1 || always_reduce)
        return reduce_splits(t, ns, a->F, a->ncols, a->dw, a->dw_stride, a->accumulate, a->F, 0, 1,
                             (cudaStream_t)stream);
      return 0;
    }
  }
  p.N = a->N; p.rows_out = a->rows_out; p.ncols = a->ncols;
  p.total_rows = (long long)a->N * a->rows_out;
  p.src = a->src; p.F = a->F; p.src_rows = a->src_rows; p.src_stride = a->src_stride;
  p.g = a->g;
  p.vec = (a->F % 4 == 0) && (a->src_stride % 4 == 0) && aligned16(a->src);
  p.gvec = (a->ncols % 4 == 0) && aligned16(a->g);
  const int ftiles = (a->F + DW_BF - 1) / DW_BF, ctiles = (a->ncols + DW_BC - 1) / DW_BC;
  const long long tiles = (long long)ftiles * ctiles;
  long long nsplit = (4LL * t->sm_count + tiles - 1) / tiles;
  const long long max_by_rows = (p.total_rows + 255) / 256;
  if (nsplit > max_by_rows) nsplit = max_by_rows;
  const long long per = (long long)a->F * a->ncols * (long long)sizeof(float);
  if (nsplit > 1 && nsplit * per > t->workspace_bytes) nsplit = t->workspace_bytes / per;
  if (nsplit < 1) nsplit = 1;
  long long rps = (p.total_rows + nsplit - 1) / nsplit;
  rps = (rps + DW_BR - 1) / DW_BR * DW_BR;
  nsplit = (p.total_rows + rps - 1) / rps;
  p.rows_per_split = rps; p.nsplit = (int)nsplit; p.accumulate = a->accumulate;
  cudaStream_t st = (cudaStream_t)stream;
  if (nsplit == 1) { p.out = a->dw; p.out_rs = a->dw_stride; }
  else { p.out = (float*)t->workspace; p.out_rs = a->ncols; }
  dim3 grid(ftiles, ctiles, (unsigned)nsplit);
  ellconv_dw_kernel<<<grid, NT, 0, st>>>(p);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  if (nsplit > 1)
    return reduce_splits(t, (int)nsplit, a->F, a->ncols, a->dw, a->dw_stride, a->accumulate, a->F, 0, 1, st);
  return 0;
}

extern "C" int cape_colsum(cape_topology* t, const float* g, int g_stride, int N, int rows, int ncols, const int* ops,
                           int nops, float* out, void* stream) {
  CAPE_REQUIRE(t && g && out, "null pointer");
  CAPE_REQUIRE(nops >= 1 && nops <= CS_MAXOPS, "nops out of range");
  CAPE_REQUIRE(N > 0 && rows > 0 && ncols > 0, "empty problem");
  ColsumParams p{};
  CAPE_REQUIRE(g_stride >= ncols, "bad g_stride");
  p.g = g; p.N = N; p.rows = rows; p.ncols = ncols; p.nops = nops; p.out = out; p.gs = g_stride;
  for (int j = 0; j < nops; ++j) {
    const int op = ops ? ops[j] : -1;
    if (op < 0) { p.coef[j] = nullptr; continue; }
    CAPE_REQUIRE(op < (int)t->ops.size(), "operator id out of range");
    CAPE_REQUIRE(t->ops[op].rows_out == rows, "colsum: operator rows mismatch");
    p.coef[j] = t->ops[op].rowsum;
  }
  p.vec = (ncols % 4 == 0) && (g_stride % 4 == 0) && ncols <= 512 && (256 % (ncols / 4) == 0) && aligned16(g);
  int rblocks = (4 * t->sm_count + N - 1) / N;
  if (rblocks < 1) rblocks = 1;
  int rpb = (rows + rblocks - 1) / rblocks;
  if (rpb < 64) rpb = 64;
  rblocks = (rows + rpb - 1) / rpb;
  p.rows_per_block = rpb;
  CAPE_REQUIRE(N <= 65535, "grid too large");
  dim3 grid(rblocks, N);
  colsum_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(p);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}
