// The conv epilogues (CAPE_EPI_*, CAPE_ACT_*) and the condition broadcast, defined once for every kernel that runs
// them: ellconv_kernel, conv_wg_kernel, apply_kernel, thin_fwd_kernel and thinout_combine_kernel.  The kernels keep
// their own loads and stores, which differ in width; what an output element is, given its loaded inputs, is decided
// here.
#pragma once
#include "common.cuh"

namespace cape {

struct EpiParams {
  int epilogue, act;
  float alpha;
  const float* bias;
  int bias_per_row;
  const float* aux;
  float* out;
  float* out2;
};

__host__ __device__ __forceinline__ bool epi_reads_aux(int epilogue) {
  return epilogue == CAPE_EPI_SLOPE || epilogue == CAPE_EPI_DUALMASK || epilogue == CAPE_EPI_TANHGRAD;
}

// The tanh epilogues (b1tanh) are compiled only into instantiations of their own (template flag TANH) in the kernels
// that unroll the epilogue over many columns: as a run-time branch the precise tanhf slowed the other activations.
inline bool needs_tanh(const EpiParams& e) { return e.act == CAPE_ACT_TANH || e.epilogue == CAPE_EPI_TANHGRAD; }

// The epilogue of a cape_conv_args or cape_apply_args, checked.  dual: the call has a second accumulator.
template <class Args>
int fill_epilogue(const Args* a, bool dual, EpiParams* e) {
  CAPE_REQUIRE(a->epilogue >= CAPE_EPI_LINEAR && a->epilogue <= CAPE_EPI_TANHGRAD, "unknown epilogue");
  CAPE_REQUIRE(a->act >= CAPE_ACT_NONE && a->act <= CAPE_ACT_TANH, "unknown activation");
  CAPE_REQUIRE(a->epilogue != CAPE_EPI_AFFINE || dual, "AFFINE epilogue needs a second accumulator");
  CAPE_REQUIRE(!epi_reads_aux(a->epilogue) || a->aux, "epilogue needs aux");
  *e = EpiParams{a->epilogue, a->act, a->alpha, a->bias, a->bias_per_row, a->aux, a->out, a->out2};
  return 0;
}

// Samples a tile of `rows` consecutive output rows can touch (bound for the condition staging buffers).
inline long long max_tile_samples(long long rows, int rows_out) { return (rows - 1) / rows_out + 2; }

// TANH = false compiles tanh out: CAPE_ACT_TANH then passes v through.
template <bool TANH>
__device__ __forceinline__ float activate(float v, int act, float alpha) {
  if (act == CAPE_ACT_LEAKY) return v > 0.f ? v : alpha * v;
  if (act == CAPE_ACT_RELU) return fmaxf(v, 0.f);
  if (TANH && act == CAPE_ACT_TANH) return tanhf(v);
  return v;
}

// W output elements from their accumulators v0 and v1 (v1 = 0 without a second one), bias (0 unless LINEAR) and aux
// (0 unless epi_reads_aux): o1 goes to out, and o2 to out2 when it returns true.  TANH = false compiles TANHGRAD out.
template <bool TANH, int W>
__device__ __forceinline__ bool apply_epilogue(const EpiParams& e, const float (&v0)[W], const float (&v1)[W],
                                               const float (&bias)[W], const float (&aux)[W], float (&o1)[W],
                                               float (&o2)[W]) {
  if (e.epilogue == CAPE_EPI_LINEAR) {
#pragma unroll
    for (int j = 0; j < W; ++j) o1[j] = activate<TANH>(v0[j] + bias[j], e.act, e.alpha);
    return false;
  }
  if (e.epilogue == CAPE_EPI_AFFINE) {
#pragma unroll
    for (int j = 0; j < W; ++j) {
      const float rg = fmaxf(v0[j], 0.f);
      o1[j] = v1[j] + rg;
      o2[j] = rg;
    }
    return e.out2 != nullptr;
  }
  if (e.epilogue == CAPE_EPI_SLOPE) {
#pragma unroll
    for (int j = 0; j < W; ++j) o1[j] = v0[j] * (aux[j] > 0.f ? 1.f : e.alpha);
    return false;
  }
  if (TANH && e.epilogue == CAPE_EPI_TANHGRAD) {
#pragma unroll
    for (int j = 0; j < W; ++j) o1[j] = v0[j] * (1.f - aux[j] * aux[j]);
    return false;
  }
#pragma unroll
  for (int j = 0; j < W; ++j) {   // DUALMASK
    o1[j] = v0[j];
    o2[j] = aux[j] > 0.f ? v0[j] : 0.f;
  }
  return e.out2 != nullptr;
}

// ---- condition broadcast ------------------------------------------------------------------------------------------
// A slot is a condition weight matrix Wc_slot[j, c] = slot_w[slot][j * slot_ws[slot] + c] (j < C).  Its term in output
// row r of sample n is rowsum(op)[r] * q_slot(n)[c] with q_slot(n) = cond[n, :] . Wc_slot, op the slot's operator.

// Stages q_slot(n_first + s)[col0 + c] for s < S, every slot and c < width (0 past ncols) at
// qs[(s * nslots + slot) * width + c] (cond_vec), with threads tid, tid + nthreads, ...
// P: a parameter block with cond, C, nslots, slot_w and slot_ws.  UNROLL: the dot products' unroll factor (loads in
// flight); the kernels that stage once per CTA keep their registers for the main loop with 4.
template <int UNROLL, class P>
__device__ __forceinline__ void stage_cond(const P& p, float* qs, int n_first, int S, int col0, int width, int ncols,
                                           int tid, int nthreads) {
  const int total = S * p.nslots * width;
  for (int o = tid; o < total; o += nthreads) {
    const int c = o % width, slot = (o / width) % p.nslots, s = o / (width * p.nslots);
    float q = 0.f;
    if (col0 + c < ncols) {
      const float* y = p.cond + (size_t)(n_first + s) * p.C;
      const float* wc = p.slot_w[slot] + col0 + c;
      const int ws = p.slot_ws[slot];
#pragma unroll UNROLL
      for (int j = 0; j < p.C; ++j) q = fmaf(__ldg(y + j), __ldg(wc + (size_t)j * ws), q);
    }
    qs[o] = q;
  }
}

// the staged q of a slot for the tile's s-th sample
__device__ __forceinline__ const float* cond_vec(const float* qs, int s, int slot, int nslots, int width) {
  return qs + ((size_t)s * nslots + slot) * width;
}

// rowsum(op)[r], the factor of a slot's q in output row r (1 for the identity): acc = fmaf(coef, q, acc) in slot order
__device__ __forceinline__ float cond_coef(const OpView& op, int r) { return op.rowsum ? __ldg(op.rowsum + r) : 1.f; }

}  // namespace cape
