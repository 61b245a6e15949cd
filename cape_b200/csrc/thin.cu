// Kernels for the "thin-input" layers: sources with <= 4 channels (the 3-channel mesh offsets entering the encoder
// and the discriminator, the 3-channel output gradient entering the decoder's backward pass, the 1-channel logit
// gradient).  These layers have almost no arithmetic (K*Fin <= 32 multiply-adds per output), so they are pure
// HBM problems: read a few MB, write/read the wide [N, rows, 32..128] tensor once.  The generic tiled kernels
// spend their time on padded reductions and scalar gathers here; these two do the Chebyshev basis on the thin
// side in registers/shared memory and stream the wide side with fully coalesced accesses.
//   thin_fwd_kernel : cape_cheb_fwd when every term has F <= 4   (lib/models.py:69-109 for enc/disc conv1, and the
//                     data-gradient of the decoder's output conv / the discriminator's prediction map)
//   thin_dw_kernel  : cape_cheb_dw  when F <= 4                  (weight gradient of the same layers)
// and the "thin-output" layers (<= 4 output columns: the decoder's 3-channel output conv, the 1-channel prediction
// map, the data gradient of the discriminator's first conv):  contract first, gather afterwards --
//   thinout_project_kernel : z[n, r', (t, c)] = sum_f src[n, r', f] W_t[f, c]      one coalesced pass over the wide source
//   thinout_combine_kernel : out[n, r, c] = sum_t sum_j op_t[r, j] z[n, idx, (t, c)] (+condition, bias, activation)
// so the operators act on 16-byte rows instead of F-wide ones.
#include "common.cuh"
#include "ellconv_params.cuh"

namespace cape {

namespace {

constexpr int TH_ROWS = 128;      // output rows per block (forward)
constexpr int TH_MAXKF = 32;      // total thin channels over all terms
constexpr int TH_MAXCOLS = 128;
constexpr int TH_QS = 1024;       // condition vectors: samples-in-tile x slots x ncols

// thin gather: out[f] = sum_j w[r,j] * src[n, idx[r,j], f]  for f < F (F <= 4), four taps per table fetch
__device__ __forceinline__ void thin_gather(const OpView& op, int r, const float* base, size_t stride, int F,
                                            float (&v)[4]) {
  v[0] = v[1] = v[2] = v[3] = 0.f;
  if (op.idx == nullptr) {
    const float* s = base + (size_t)r * stride;
#pragma unroll
    for (int f = 0; f < 4; ++f)
      if (f < F) v[f] = __ldg(s + f);
    return;
  }
  const int4* ip = reinterpret_cast<const int4*>(op.idx + (size_t)r * op.width);
  const float4* wp = reinterpret_cast<const float4*>(op.w + (size_t)r * op.width);
  const int nb = op.width >> 2;
  for (int b = 0; b < nb; ++b) {
    const int4 id = __ldg(ip + b);
    if (id.x < 0) break;
    const float4 ww = __ldg(wp + b);
    const int ids[4] = {id.x, max(id.y, 0), max(id.z, 0), max(id.w, 0)};
    const float ws[4] = {ww.x, ww.y, ww.z, ww.w};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float* s = base + (size_t)ids[u] * stride;
#pragma unroll
      for (int f = 0; f < 4; ++f)
        if (f < F) v[f] = fmaf(ws[u], __ldg(s + f), v[f]);
    }
  }
}

// TANH: the tanh epilogues (needs_tanh)
template <bool TANH>
__global__ void __launch_bounds__(256) thin_fwd_kernel(const __grid_constant__ ConvParams p, int KF, int vec4) {
  __shared__ float Bs[TH_ROWS][TH_MAXKF + 1];
  __shared__ __align__(16) float Ws[TH_MAXKF * TH_MAXCOLS];
  __shared__ __align__(16) float qs[TH_QS];
  __shared__ int s_n[TH_ROWS], s_r[TH_ROWS];
  __shared__ int s_off[CAPE_MAX_TERMS];

  const int tid = threadIdx.x;
  const long long row0 = (long long)blockIdx.x * TH_ROWS;
  const int ncols = p.ncols;
  if (tid < TH_ROWS) {
    const long long R = row0 + tid;
    if (R < p.total_rows) { s_n[tid] = (int)(R / p.rows_out); s_r[tid] = (int)(R % p.rows_out); }
    else { s_n[tid] = -1; s_r[tid] = 0; }
  }
  if (tid == 0) {
    int o = 0;
    for (int t = 0; t < p.nterms; ++t) { s_off[t] = o; o += p.terms[t].F; }
  }
  // weights: Ws[q][c] with q running over (term, f)
  for (int e = tid; e < KF * ncols; e += 256) {
    const int q = e / ncols, c = e % ncols;
    int t = 0, o = 0;
    while (t + 1 < p.nterms && q >= o + p.terms[t].F) { o += p.terms[t].F; ++t; }
    Ws[e] = __ldg(p.terms[t].w + (size_t)(q - o) * p.terms[t].w_stride + c);
  }
  __syncthreads();

  // ---- phase 1: Chebyshev basis of the thin source, one (row, term) item per thread iteration
  for (int item = tid; item < TH_ROWS * p.nterms; item += 256) {
    const int row = item % TH_ROWS, t = item / TH_ROWS;
    const TermDev& tm = p.terms[t];
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    const int n = s_n[row];
    if (n >= 0) thin_gather(tm.op, s_r[row], tm.src + (size_t)n * tm.src_rows * tm.src_stride, (size_t)tm.src_stride, tm.F, v);
    const int o = s_off[t];
#pragma unroll
    for (int f = 0; f < 4; ++f)
      if (f < tm.F) Bs[row][o + f] = v[f];
  }
  // ---- condition broadcast vectors
  const int n_first = s_n[0];
  if (p.nslots > 0) {
    int n_last = n_first;
    for (int i = TH_ROWS - 1; i > 0; --i)
      if (s_n[i] >= 0) { n_last = s_n[i]; break; }
    stage_cond<16>(p, qs, n_first, n_last - n_first + 1, 0, ncols, ncols, tid, 256);
  }
  __syncthreads();
  const EpiParams& e = p.epi;

  // ---- phase 2: outputs, coalesced along the columns -- four columns per thread when everything is 16-byte aligned
  if (vec4) {
    const int nc4 = ncols >> 2;
    for (int o = tid; o < TH_ROWS * nc4; o += 256) {
      const int row = o / nc4, c = (o % nc4) * 4;
      const int n = s_n[row];
      if (n < 0) continue;
      const int r = s_r[row];
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int q = 0; q < KF; ++q) fma4(acc, Bs[row][q], *reinterpret_cast<const float4*>(&Ws[q * ncols + c]));
      for (int slot = 0; slot < p.nslots; ++slot)
        fma4(acc, cond_coef(p.terms[p.slot_term[slot]].op, r),
             *reinterpret_cast<const float4*>(cond_vec(qs, n - n_first, slot, p.nslots, ncols) + c));
      const size_t oi = (size_t)(row0 + row) * ncols + c;
      float v0[4] = {acc.x, acc.y, acc.z, acc.w}, zero[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
      float ax[4] = {0.f, 0.f, 0.f, 0.f}, o1[4], o2[4];
      if (e.epilogue == CAPE_EPI_LINEAR && e.bias != nullptr) {
        const float4 b4 = ldg4(e.bias + (e.bias_per_row ? (size_t)r * ncols : 0) + c);
        b[0] = b4.x; b[1] = b4.y; b[2] = b4.z; b[3] = b4.w;
      } else if (epi_reads_aux(e.epilogue)) {
        const float4 a4 = ldg4(e.aux + oi);
        ax[0] = a4.x; ax[1] = a4.y; ax[2] = a4.z; ax[3] = a4.w;
      }
      const bool write2 = apply_epilogue<TANH>(e, v0, zero, b, ax, o1, o2);
      *reinterpret_cast<float4*>(e.out + oi) = make_float4(o1[0], o1[1], o1[2], o1[3]);
      if (write2) *reinterpret_cast<float4*>(e.out2 + oi) = make_float4(o2[0], o2[1], o2[2], o2[3]);
    }
    return;
  }
  for (int o = tid; o < TH_ROWS * ncols; o += 256) {
    const int row = o / ncols, c = o % ncols;
    const int n = s_n[row];
    if (n < 0) continue;
    const int r = s_r[row];
    float acc = 0.f;
    for (int q = 0; q < KF; ++q) acc = fmaf(Bs[row][q], Ws[q * ncols + c], acc);
    for (int slot = 0; slot < p.nslots; ++slot)
      acc = fmaf(cond_coef(p.terms[p.slot_term[slot]].op, r), cond_vec(qs, n - n_first, slot, p.nslots, ncols)[c], acc);
    const size_t oi = (size_t)(row0 + row) * ncols + c;
    float v0[1] = {acc}, zero[1] = {0.f}, b[1] = {0.f}, ax[1] = {0.f}, o1[1], o2[1];
    if (e.epilogue == CAPE_EPI_LINEAR && e.bias != nullptr)
      b[0] = __ldg(e.bias + (e.bias_per_row ? (size_t)r * ncols : 0) + c);
    else if (epi_reads_aux(e.epilogue)) ax[0] = __ldg(e.aux + oi);
    if (apply_epilogue<TANH>(e, v0, zero, b, ax, o1, o2)) e.out2[oi] = o2[0];
    e.out[oi] = o1[0];
  }
}

constexpr int TD_MAXOPS = 4;
constexpr int TD_MAXKF = 16;     // (operators) x (thin channels) accumulated in one pass over g

struct ThinDwParams {
  int rows_out, ncols, F, src_rows, src_stride, nops;
  long long total_rows, rows_per_block;
  const float* src;
  OpView op[TD_MAXOPS];
  const float* g;
  float* out;      // partial sums [gridDim.x, nops * F, ncols]
};

constexpr int TD_CHUNK = 256;

// dW of ALL the polynomial terms of a thin-input layer in one pass over the wide gradient g: the basis rows
// B[r, (op, f)] (<= 16 values) are built in shared memory 256 rows at a time, then every thread owns four columns of g
// (one 16-byte load per row) and accumulates its [KF x 4] block in registers.
template <int KF>
__global__ void __launch_bounds__(256) thin_dw_kernel(const __grid_constant__ ThinDwParams p) {
  __shared__ float Bs[TD_CHUNK][KF + 1];
  __shared__ float4 red[256];
  const int tid = threadIdx.x;
  const int ncols = p.ncols;
  const int tpr = ncols >> 2;                 // threads per row (ncols in {32, 64, 128, 256})
  const int RG = 256 / tpr;                   // rows in flight
  const int c = (tid % tpr) * 4, rg = tid / tpr;
  const long long rbeg = (long long)blockIdx.x * p.rows_per_block;
  const long long rend = min(p.total_rows, rbeg + p.rows_per_block);
  float4 acc[KF];
#pragma unroll
  for (int q = 0; q < KF; ++q) acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long rb = rbeg; rb < rend; rb += TD_CHUNK) {
    for (int item = tid; item < TD_CHUNK * p.nops; item += 256) {
      const int row = item % TD_CHUNK, j = item / TD_CHUNK;
      const long long R = rb + row;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (R < rend) {
        const int n = (int)(R / p.rows_out), r = (int)(R % p.rows_out);
        thin_gather(p.op[j], r, p.src + (size_t)n * p.src_rows * p.src_stride, (size_t)p.src_stride, p.F, v);
      }
#pragma unroll
      for (int f = 0; f < 4; ++f)
        if (j * p.F + f < KF && f < p.F) Bs[row][j * p.F + f] = v[f];
    }
    __syncthreads();
    const int lim = (int)min((long long)TD_CHUNK, rend - rb);
#pragma unroll 2
    for (int r = rg; r < lim; r += RG) {
      const float4 gv = ldg4(p.g + (size_t)(rb + r) * ncols + c);
#pragma unroll
      for (int q = 0; q < KF; ++q) fma4(acc[q], Bs[r][q], gv);
    }
    __syncthreads();
  }
  // reduce the row groups (fixed order) and write this block's partial sums
  const int nq = p.nops * p.F;
#pragma unroll
  for (int q = 0; q < KF; ++q) {
    if (q < nq) {
      red[tid] = acc[q];
      __syncthreads();
      if (rg == 0) {
        float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int k = 0; k < RG; ++k) {
          const float4 t4 = red[k * tpr + tid];
          s4.x += t4.x; s4.y += t4.y; s4.z += t4.z; s4.w += t4.w;
        }
        *reinterpret_cast<float4*>(p.out + ((size_t)blockIdx.x * nq + q) * ncols + c) = s4;
      }
      __syncthreads();
    }
  }
}

// ---- thin output -------------------------------------------------------------------------------------------------
constexpr int TO_MAXT = 4;        // terms
constexpr int TO_ZW = 16;         // floats per z row: 4 terms x 4 columns

struct ThinOutW {
  const float* w[TO_MAXT];
  int ws[TO_MAXT];
};

__global__ void __launch_bounds__(256) thinout_project_kernel(const float* __restrict__ src, int F, int src_stride,
                                                              long long nrows, int nterms, int ncols,
                                                              const __grid_constant__ ThinOutW wt, float* __restrict__ z) {
  // Ws[(t*4 + c)][f], one warp per source row, lanes over f (float4), 16 running sums per lane, butterfly reduction
  extern __shared__ __align__(16) float Ws[];
  for (int e = threadIdx.x; e < F * TO_ZW; e += 256) {
    const int q = e / F, f = e % F, t = q >> 2, c = q & 3;
    Ws[e] = (t < nterms && c < ncols) ? __ldg(wt.w[t] + (size_t)f * wt.ws[t] + c) : 0.f;
  }
  __syncthreads();
  // lpr lanes share a source row (F / 4 of them are busy; narrow sources put 2 or 4 rows on a warp)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lpr = F >= 128 ? 32 : (F >= 64 ? 16 : 8), rpw = 32 / lpr;
  const int sub = lane / lpr, l = lane % lpr;
  const int nq = nterms * 4;
  for (long long R0 = ((long long)blockIdx.x * 8 + warp) * rpw; R0 < nrows; R0 += (long long)gridDim.x * 8 * rpw) {
    const long long R = R0 + sub;
    float acc[TO_ZW];
#pragma unroll
    for (int q = 0; q < TO_ZW; ++q) acc[q] = 0.f;
    if (R < nrows) {
      const float* row = src + (size_t)R * src_stride;
      for (int f = l * 4; f < F; f += lpr * 4) {
        const float4 v = ldg4(row + f);
#pragma unroll
        for (int q = 0; q < TO_ZW; ++q) {
          if (q < nq) {
            const float4 w = *reinterpret_cast<const float4*>(&Ws[q * F + f]);
            acc[q] += v.x * w.x + v.y * w.y + v.z * w.z + v.w * w.w;
          }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < TO_ZW; ++q) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        if (o < lpr) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
    }
    if (R < nrows) {
#pragma unroll
      for (int g = 0; g < 4; ++g)
        if (l == g)
          *reinterpret_cast<float4*>(z + (size_t)R * TO_ZW + g * 4) =
              make_float4(acc[g * 4], acc[g * 4 + 1], acc[g * 4 + 2], acc[g * 4 + 3]);
    }
  }
}

struct ThinOutParams {
  int rows_out, src_rows, ncols, nterms;
  long long total_rows;
  OpView op[TO_MAXT];
  const float* z;
  // condition: q[n][slot][c] = cond[n,:] @ Wc_slot[:, c], scaled by rowsum(op of the slot's term)
  int nslots, C;
  int slot_term[TO_MAXT];
  const float* slot_w[TO_MAXT];
  int slot_ws[TO_MAXT];
  const float* cond;
  EpiParams epi;       // LINEAR
};

constexpr int TO_MAXS = 8;        // samples a 256-row block may touch

__global__ void __launch_bounds__(256) thinout_combine_kernel(const __grid_constant__ ThinOutParams p) {
  __shared__ float qs[TO_MAXS * TO_MAXT * 4];
  const long long R0 = (long long)blockIdx.x * 256;
  const int n_first = (int)(R0 / p.rows_out);
  if (p.nslots > 0) {
    // condition vectors of the samples in this block
    const long long rlast = min(p.total_rows, R0 + 256) - 1;
    stage_cond<4>(p, qs, n_first, (int)(rlast / p.rows_out) - n_first + 1, 0, 4, p.ncols, threadIdx.x, 256);
    __syncthreads();
  }
  const long long R = R0 + threadIdx.x;
  if (R >= p.total_rows) return;
  const int n = (int)(R / p.rows_out), r = (int)(R % p.rows_out);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const float* zb = p.z + (size_t)n * p.src_rows * TO_ZW;
  for (int t = 0; t < p.nterms; ++t) {
    const OpView& op = p.op[t];
    if (op.idx == nullptr) {
      const float4 v = ldg4(zb + (size_t)r * TO_ZW + t * 4);
      acc[0] += v.x; acc[1] += v.y; acc[2] += v.z; acc[3] += v.w;
      continue;
    }
    const int4* ip = reinterpret_cast<const int4*>(op.idx + (size_t)r * op.width);
    const float4* wp = reinterpret_cast<const float4*>(op.w + (size_t)r * op.width);
    const int nb = op.width >> 2;
    for (int b = 0; b < nb; ++b) {
      const int4 id = __ldg(ip + b);
      if (id.x < 0) break;
      const float4 ww = __ldg(wp + b);
      const float4 v0 = ldg4(zb + (size_t)id.x * TO_ZW + t * 4), v1 = ldg4(zb + (size_t)max(id.y, 0) * TO_ZW + t * 4);
      const float4 v2 = ldg4(zb + (size_t)max(id.z, 0) * TO_ZW + t * 4), v3 = ldg4(zb + (size_t)max(id.w, 0) * TO_ZW + t * 4);
      acc[0] += ww.x * v0.x + ww.y * v1.x + ww.z * v2.x + ww.w * v3.x;
      acc[1] += ww.x * v0.y + ww.y * v1.y + ww.z * v2.y + ww.w * v3.y;
      acc[2] += ww.x * v0.z + ww.y * v1.z + ww.z * v2.z + ww.w * v3.z;
      acc[3] += ww.x * v0.w + ww.y * v1.w + ww.z * v2.w + ww.w * v3.w;
    }
  }
  for (int s = 0; s < p.nslots; ++s) {
    const float coef = cond_coef(p.op[p.slot_term[s]], r);
    const float* q = cond_vec(qs, n - n_first, s, p.nslots, 4);
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[c] = fmaf(coef, q[c], acc[c]);
  }
  const EpiParams& e = p.epi;
  for (int c = 0; c < p.ncols; ++c) {
    float v = acc[c];
    if (e.bias != nullptr) v += __ldg(e.bias + (e.bias_per_row ? (size_t)r * p.ncols : 0) + c);
    e.out[(size_t)R * p.ncols + c] = activate<true>(v, e.act, e.alpha);
  }
}

}  // namespace

// returns 1 if launched, 0 if not eligible
int launch_thin_fwd(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st) {
  (void)t;
  if (dual || p.epi.epilogue == CAPE_EPI_AFFINE || p.npass > 0) return 0;   // pass-through terms: ellconv kernels
  if (p.ncols > TH_MAXCOLS || p.ncols < 16) return 0;
  int KF = 0;
  for (int i = 0; i < p.nterms; ++i) {
    if (p.terms[i].F > 4 || p.terms[i].stash != nullptr) return 0;
    KF += p.terms[i].F;
  }
  if (KF > TH_MAXKF) return 0;
  if (max_tile_samples(TH_ROWS, p.rows_out) * p.nslots * p.ncols > TH_QS) return 0;
  for (int s = 0; s < p.nslots; ++s)
    if (p.slot_acc[s] != 0) return 0;
  const unsigned grid = (unsigned)((p.total_rows + TH_ROWS - 1) / TH_ROWS);
  const int vec4 = (p.ncols % 4 == 0) && p.ovec && (p.epi.bias == nullptr || aligned16(p.epi.bias));
  if (needs_tanh(p.epi)) thin_fwd_kernel<true><<<grid, 256, 0, st>>>(p, KF, vec4);
  else thin_fwd_kernel<false><<<grid, 256, 0, st>>>(p, KF, vec4);
  CAPE_CHECK_CUDA(cudaGetLastError());
  count_launches(1);
  return 1;
}

// returns 1 if launched (partials [*nsplit_out, nops * F, ncols] in the workspace), 0 if not eligible
int launch_thin_dw(const cape_topology* t, const cape_dw_args* a, const OpView* ops, int nops, int* nsplit_out,
                   cudaStream_t st) {
  if (a->F > 4 || nops < 1 || nops > TD_MAXOPS || nops * a->F > TD_MAXKF) return 0;
  if (!(a->ncols == 32 || a->ncols == 64 || a->ncols == 128 || a->ncols == 256) || !aligned16(a->g)) return 0;
  ThinDwParams p{};
  p.rows_out = a->rows_out; p.ncols = a->ncols; p.F = a->F; p.src_rows = a->src_rows; p.src_stride = a->src_stride;
  p.total_rows = (long long)a->N * a->rows_out;
  p.src = a->src; p.g = a->g; p.nops = nops;
  for (int j = 0; j < nops; ++j) p.op[j] = ops[j];
  const int nq = nops * a->F;
  // one full wave: the register count of thin_dw_kernel<KF> admits 4 / 3 / 2 / 2 CTAs per SM for KF = 4 / 8 / 12 / 16
  // (with 4 x SMs blocks the KF = 8 kernel ran 1.3 waves of three 256-row chunks: two rounds where 4 chunks in one do)
  const int resident = nq <= 4 ? 4 : (nq <= 8 ? 3 : 2);
  long long nblk = (g_tuning[17] == 1 ? 4LL : (long long)resident) * t->sm_count;
  const long long max_by_rows = (p.total_rows + TD_CHUNK - 1) / TD_CHUNK;
  if (nblk > max_by_rows) nblk = max_by_rows;
  const long long per = (long long)nq * a->ncols * (long long)sizeof(float);
  if (nblk * per > t->workspace_bytes) nblk = t->workspace_bytes / per;
  if (nblk < 1) return 0;
  long long rpb = (p.total_rows + nblk - 1) / nblk;
  rpb = (rpb + TD_CHUNK - 1) / TD_CHUNK * TD_CHUNK;
  nblk = (p.total_rows + rpb - 1) / rpb;
  p.rows_per_block = rpb;
  p.out = (float*)t->workspace;
  if (nq <= 4) thin_dw_kernel<4><<<(unsigned)nblk, 256, 0, st>>>(p);
  else if (nq <= 8) thin_dw_kernel<8><<<(unsigned)nblk, 256, 0, st>>>(p);
  else if (nq <= 12) thin_dw_kernel<12><<<(unsigned)nblk, 256, 0, st>>>(p);
  else thin_dw_kernel<16><<<(unsigned)nblk, 256, 0, st>>>(p);
  CAPE_CHECK_CUDA(cudaGetLastError());
  count_launches(1);
  *nsplit_out = (int)nblk;
  return 1;
}

// thin-output conv: 1 = launched (z lives in the topology workspace), 0 = not eligible
int launch_thinout_fwd(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st) {
  if (dual || p.epi.epilogue != CAPE_EPI_LINEAR || p.ncols > 4 || p.nterms > TO_MAXT || p.npass > 0 || g_tuning[7] == 1)
    return 0;
  const TermDev& t0 = p.terms[0];
  if (!t0.vec || t0.F < 32 || t0.F % 4 != 0 || t0.F > 512) return 0;
  for (int i = 0; i < p.nterms; ++i) {
    const TermDev& tm = p.terms[i];
    if (tm.src != t0.src || tm.F != t0.F || tm.src_rows != t0.src_rows || tm.src_stride != t0.src_stride ||
        tm.stash != nullptr)
      return 0;
  }
  if (p.nslots > TO_MAXT || (p.nslots > 0 && max_tile_samples(256, p.rows_out) > TO_MAXS)) return 0;
  for (int s = 0; s < p.nslots; ++s)
    if (p.slot_acc[s] != 0) return 0;
  const long long nsrc = (long long)p.N * t0.src_rows;
  const size_t zbytes = (size_t)nsrc * TO_ZW * sizeof(float);
  if (zbytes > (size_t)t->workspace_bytes) return 0;
  ThinOutW h{};
  for (int i = 0; i < p.nterms; ++i) { h.w[i] = p.terms[i].w; h.ws[i] = p.terms[i].w_stride; }
  float* z = reinterpret_cast<float*>(t->workspace);
  const size_t smem = (size_t)t0.F * TO_ZW * sizeof(float);
  static bool configured = false;
  if (!configured) {
    CAPE_CHECK_CUDA(cudaFuncSetAttribute(thinout_project_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 512 * TO_ZW * 4));
    configured = true;
  }
  long long blocks = (nsrc + 7) / 8;
  if (blocks > 8LL * t->sm_count) blocks = 8LL * t->sm_count;
  thinout_project_kernel<<<(unsigned)blocks, 256, smem, st>>>(
      t0.src, t0.F, t0.src_stride, nsrc, p.nterms, p.ncols, h, z);
  CAPE_CHECK_CUDA(cudaGetLastError());
  ThinOutParams q{};
  q.rows_out = p.rows_out; q.src_rows = t0.src_rows; q.ncols = p.ncols; q.nterms = p.nterms; q.total_rows = p.total_rows;
  for (int i = 0; i < p.nterms; ++i) q.op[i] = p.terms[i].op;
  q.z = z; q.nslots = p.nslots; q.C = p.C; q.cond = p.cond;
  for (int s = 0; s < p.nslots; ++s) {
    q.slot_term[s] = p.slot_term[s]; q.slot_w[s] = p.slot_w[s]; q.slot_ws[s] = p.slot_ws[s];
  }
  q.epi = p.epi;
  thinout_combine_kernel<<<(unsigned)((p.total_rows + 255) / 256), 256, 0, st>>>(q);
  CAPE_CHECK_CUDA(cudaGetLastError());
  count_launches(2);
  return 1;
}

}  // namespace cape
