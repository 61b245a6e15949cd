// cape_apply: sparse operators applied to feature rows, no contraction --
//   acc_a[n, r, c] = sum_{t: acc(t) = a} scale_t * ( sum_j op_t[r, j] * src_t[n, idx_t[r, j], c]  +  rowsum(op_t)[r] * (cond[n, :] @ wc_t)[c] )
// followed by the same epilogues as the fused conv (bias / activation, affine block, backward masks).
//
// It is the gather half of the two split forms of chebyshev5 (lib/models.py:69-103) the host uses next to the fused
// kernel:
//   contract first:  Z = X . [W_0 | W_1 | ... ] on the tensor-core kernel (ellconv_tc.cu), then
//                    out = epi( sum_k op_k Z_k )                 -- the operators touch Fout-wide rows instead of Fin-wide
//                    ones, and the contraction runs over the (fewer) rows of the coarse level when op_k un-pools;
//   basis first:     B_k = op_k X (this kernel, written where the weight gradient wants it anyway), then the
//                    contraction of plain tensors on the tensor-core kernel.
// A pure SIMT kernel: one float4 column group of one row per thread, two rows in flight per thread (eight independent
// neighbour-row loads), no shared-memory tiles -- so all 64 warps of an SM are resident, the L1 is ~200 KB and a CTA's
// 64 consecutive rows re-hit each other's one-rings in it.  Bound: L2 -> SM bandwidth of the neighbour rows.
#include "common.cuh"
#include "ellconv_params.cuh"

namespace cape {

namespace {

constexpr int AP_THREADS = 256;
constexpr int AP_ROWS = 128;           // rows per CTA (experiment knob 10 overrides)
constexpr int AP_QS = 3072;            // floats of condition vectors per CTA

struct ApTerm {
  const float* src;
  OpView op;
  int src_rows, src_stride, acc;
  float scale;
  int slot;                            // index of its condition vector, -1: none
};

struct ApParams {
  int N, rows_out, ncols, nterms, tpr, rpp;     // threads per row, rows per pass
  int rows_cta;                                 // rows per CTA
  long long total_rows;
  ApTerm terms[CAPE_MAX_TERMS];
  int nslots;
  const float* slot_w[CAPE_MAX_TERMS];
  int slot_ws[CAPE_MAX_TERMS];
  const float* cond;
  int C;
  int epilogue, act;
  float alpha;
  const float* bias;
  int bias_per_row;
  const float* aux;
  float* out;
  float* out2;
  int out_stride;
  long long term_stride;               // > 0: "separate" mode, term t is written on its own to out + t * term_stride
};

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void f4_axpy(float4& a, float s, const float4& x) {
  a.x = fmaf(s, x.x, a.x); a.y = fmaf(s, x.y, a.y); a.z = fmaf(s, x.z, a.z); a.w = fmaf(s, x.w, a.w);
}

__device__ __forceinline__ void ap_advance(int& r, int& n, int by, int rows) {
  r += by;
  while (r >= rows) { r -= rows; ++n; }
}

template <bool DUAL>
__device__ __forceinline__ void ap_store(const ApParams& p, long long R, int r, int c, float4 a0, float4 a1) {
  const size_t o = (size_t)R * p.out_stride + c;
  float v0[4] = {a0.x, a0.y, a0.z, a0.w}, v1[4] = {a1.x, a1.y, a1.z, a1.w}, o1[4], o2[4];
  bool write2 = false;
  if (p.epilogue == CAPE_EPI_LINEAR) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v = v0[j];
      if (p.bias != nullptr) v += __ldg(p.bias + (p.bias_per_row ? (size_t)r * p.ncols : 0) + c + j);
      if (p.act == CAPE_ACT_LEAKY) v = v > 0.f ? v : p.alpha * v;
      else if (p.act == CAPE_ACT_RELU) v = fmaxf(v, 0.f);
      o1[j] = v;
    }
  } else if (p.epilogue == CAPE_EPI_AFFINE) {
    write2 = p.out2 != nullptr;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float rg = fmaxf(v0[j], 0.f);
      o1[j] = (DUAL ? v1[j] : 0.f) + rg;
      o2[j] = rg;
    }
  } else {
    const float4 ax = ldg4(p.aux + (size_t)R * p.ncols + c);
    const float a[4] = {ax.x, ax.y, ax.z, ax.w};
    if (p.epilogue == CAPE_EPI_SLOPE) {
#pragma unroll
      for (int j = 0; j < 4; ++j) o1[j] = v0[j] * (a[j] > 0.f ? 1.f : p.alpha);
    } else {
      write2 = p.out2 != nullptr;
#pragma unroll
      for (int j = 0; j < 4; ++j) { o1[j] = v0[j]; o2[j] = a[j] > 0.f ? v0[j] : 0.f; }
    }
  }
  *reinterpret_cast<float4*>(p.out + o) = make_float4(o1[0], o1[1], o1[2], o1[3]);
  if (write2) *reinterpret_cast<float4*>(p.out2 + o) = make_float4(o2[0], o2[1], o2[2], o2[3]);
}

template <bool DUAL>
__global__ void __launch_bounds__(AP_THREADS, 3) apply_kernel(const __grid_constant__ ApParams p) {
  __shared__ __align__(16) float qs[AP_QS];
  const int AP_R = p.rows_cta;
  const long long R0 = (long long)blockIdx.x * AP_R;
  const int n_first = (int)(R0 / p.rows_out);
  if (p.nslots > 0) {
    // condition vectors of the samples this CTA touches: q[s][slot][c] = cond[n_first + s, :] @ wc_slot[:, c]
    const long long rlast = min(p.total_rows, R0 + AP_R) - 1;
    const int S = (int)(rlast / p.rows_out) - n_first + 1;
    const int total = S * p.nslots * p.ncols;
    for (int o = threadIdx.x; o < total; o += AP_THREADS) {
      const int c = o % p.ncols, slot = (o / p.ncols) % p.nslots, s = o / (p.ncols * p.nslots);
      const float* y = p.cond + (size_t)(n_first + s) * p.C;
      const float* wc = p.slot_w[slot] + c;
      float q = 0.f;
      for (int j = 0; j < p.C; ++j) q = fmaf(__ldg(y + j), __ldg(wc + (size_t)j * p.slot_ws[slot]), q);
      qs[o] = q;
    }
    __syncthreads();
  }
  const int lr = threadIdx.x / p.tpr, c = (threadIdx.x % p.tpr) * 4;
  if (lr >= p.rpp) return;
  // (sample, vertex) of the thread's first row by one division, of the following rows by stepping: a 64-bit division
  // per row was a quarter of the loop's instructions
  const int step = 2 * p.rpp;
  int na = (int)((R0 + lr) / p.rows_out), ra = (int)((R0 + lr) - (long long)na * p.rows_out);
  for (int base = lr; base < AP_R; base += step, ap_advance(ra, na, step, p.rows_out)) {
    const long long Ra = R0 + base, Rb = Ra + p.rpp;
    if (Ra >= p.total_rows) break;
    const bool vb = (base + p.rpp < AP_R) && Rb < p.total_rows;
    int nb = na, rb = ra;
    if (vb) ap_advance(rb, nb, p.rpp, p.rows_out);
    float4 a0 = f4_zero(), a1 = f4_zero(), b0 = f4_zero(), b1 = f4_zero();
    for (int t = 0; t < p.nterms; ++t) {
      const ApTerm& tm = p.terms[t];
      const float* pa = tm.src + (size_t)na * tm.src_rows * tm.src_stride + c;
      const float* pb = tm.src + (size_t)nb * tm.src_rows * tm.src_stride + c;
      float4 ta = f4_zero(), tb = f4_zero();
      if (tm.op.idx == nullptr) {
        ta = ldg4(pa + (size_t)ra * tm.src_stride);
        tb = ldg4(pb + (size_t)rb * tm.src_stride);
      } else {
        ell_gather4_pair(tm.op, ra, rb, pa, pb, (size_t)tm.src_stride, ta, tb);
      }
      if (tm.slot >= 0) {
        const float ca = tm.op.rowsum ? __ldg(tm.op.rowsum + ra) : 1.f, cb = tm.op.rowsum ? __ldg(tm.op.rowsum + rb) : 1.f;
        const float4 qa = *reinterpret_cast<const float4*>(qs + ((size_t)(na - n_first) * p.nslots + tm.slot) * p.ncols + c);
        const float4 qb = *reinterpret_cast<const float4*>(qs + ((size_t)(nb - n_first) * p.nslots + tm.slot) * p.ncols + c);
        f4_axpy(ta, ca, qa);
        f4_axpy(tb, cb, qb);
      }
      if (p.term_stride > 0) {
        // separate mode (the K basis tensors of a layer in one launch): no summation, no epilogue
        float* o = p.out + (size_t)t * p.term_stride;
        *reinterpret_cast<float4*>(o + (size_t)Ra * p.out_stride + c) =
            make_float4(tm.scale * ta.x, tm.scale * ta.y, tm.scale * ta.z, tm.scale * ta.w);
        if (vb)
          *reinterpret_cast<float4*>(o + (size_t)Rb * p.out_stride + c) =
              make_float4(tm.scale * tb.x, tm.scale * tb.y, tm.scale * tb.z, tm.scale * tb.w);
        continue;
      }
      if (DUAL && tm.acc == 1) { f4_axpy(a1, tm.scale, ta); f4_axpy(b1, tm.scale, tb); }
      else { f4_axpy(a0, tm.scale, ta); f4_axpy(b0, tm.scale, tb); }
    }
    if (p.term_stride > 0) continue;
    ap_store<DUAL>(p, Ra, ra, c, a0, a1);
    if (vb) ap_store<DUAL>(p, Rb, rb, c, b0, b1);
  }
}

}  // namespace

}  // namespace cape

using namespace cape;

extern "C" int cape_apply(cape_topology* t, const cape_apply_args* a, void* stream) {
  CAPE_REQUIRE(t && a, "null handle/args");
  CAPE_REQUIRE(a->N > 0 && a->rows_out > 0 && a->ncols > 0, "empty problem");
  CAPE_REQUIRE(a->nterms >= 1 && a->nterms <= CAPE_MAX_TERMS, "nterms out of range");
  CAPE_REQUIRE(a->out != nullptr, "out is null");
  CAPE_REQUIRE(a->ncols % 4 == 0 && a->ncols <= 4 * AP_THREADS, "cape_apply needs ncols % 4 == 0 and ncols <= 1024");
  CAPE_REQUIRE(a->epilogue >= CAPE_EPI_LINEAR && a->epilogue <= CAPE_EPI_DUALMASK, "unknown epilogue");
  ApParams p{};
  p.N = a->N; p.rows_out = a->rows_out; p.ncols = a->ncols; p.nterms = a->nterms;
  p.total_rows = (long long)a->N * a->rows_out;
  p.tpr = a->ncols / 4;
  p.rows_cta = (g_tuning[10] >= 16 && g_tuning[10] <= 1024) ? g_tuning[10] : AP_ROWS;
  p.rpp = AP_THREADS / p.tpr;
  if (p.rpp > p.rows_cta / 2) p.rpp = p.rows_cta / 2;
  p.out_stride = a->out_stride > 0 ? a->out_stride : a->ncols;
  CAPE_REQUIRE(p.out_stride >= a->ncols && p.out_stride % 4 == 0 && aligned16(a->out) && (!a->out2 || aligned16(a->out2)),
               "out / out2 must be 16-byte aligned with out_stride % 4 == 0");
  bool dual = false;
  for (int i = 0; i < a->nterms; ++i) {
    const cape_apply_term& s = a->terms[i];
    ApTerm& d = p.terms[i];
    CAPE_REQUIRE(s.src && s.src_stride >= a->ncols && s.src_stride % 4 == 0 && aligned16(s.src),
                 "term needs a 16-byte aligned src with src_stride % 4 == 0 and >= ncols");
    CAPE_REQUIRE(s.acc == 0 || s.acc == 1, "acc must be 0 or 1");
    if (get_op(t, s.op, a->rows_out, s.src_rows, &d.op) != 0) return -1;
    d.src = s.src; d.src_rows = s.src_rows; d.src_stride = s.src_stride; d.acc = s.acc;
    d.scale = s.scale == 0.f ? 1.f : s.scale;
    d.slot = -1;
    if (s.acc == 1) dual = true;
    if (s.wc) {
      CAPE_REQUIRE(a->cond && a->C > 0 && s.wc_stride >= a->ncols, "condition rows without cond / bad wc_stride");
      d.slot = p.nslots;
      p.slot_w[p.nslots] = s.wc; p.slot_ws[p.nslots] = s.wc_stride; ++p.nslots;
    }
  }
  if (p.nslots > 0) {
    const long long max_samples = (p.rows_cta - 1) / a->rows_out + 2;
    CAPE_REQUIRE(max_samples * p.nslots * a->ncols <= AP_QS, "too many condition columns for the staging buffer");
  }
  p.cond = a->cond; p.C = a->C;
  p.epilogue = a->epilogue; p.act = a->act; p.alpha = a->alpha;
  p.bias = a->bias; p.bias_per_row = a->bias_per_row; p.aux = a->aux;
  p.out = a->out; p.out2 = a->out2;
  p.term_stride = a->term_stride;
  if (a->term_stride != 0) {
    CAPE_REQUIRE(a->term_stride > 0 && a->term_stride % 4 == 0 && a->epilogue == CAPE_EPI_LINEAR && !a->bias &&
                 a->act == CAPE_ACT_NONE && p.nslots == 0 && !dual,
                 "separate outputs (term_stride) take plain terms: LINEAR epilogue, no bias / activation / condition");
  }
  if (a->epilogue == CAPE_EPI_SLOPE || a->epilogue == CAPE_EPI_DUALMASK) {
    CAPE_REQUIRE(a->aux && aligned16(a->aux), "epilogue needs a 16-byte aligned aux");
    CAPE_REQUIRE(p.out_stride == a->ncols, "SLOPE / DUALMASK epilogues need out_stride == ncols");
  }
  const long long blocks = (p.total_rows + p.rows_cta - 1) / p.rows_cta;
  CAPE_REQUIRE(blocks < (1LL << 31), "grid too large");
  if (dual) apply_kernel<true><<<(unsigned)blocks, AP_THREADS, 0, (cudaStream_t)stream>>>(p);
  else apply_kernel<false><<<(unsigned)blocks, AP_THREADS, 0, (cudaStream_t)stream>>>(p);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}
