// Parameter blocks shared by the SIMT (ellconv.cu) and wgmma (ellconv_tc.cu) fused-conv kernels.
#pragma once
#include "common.cuh"

namespace cape {

constexpr int BM = 128;   // output rows per CTA
constexpr int BK = 32;    // reduction chunk
constexpr int NT = 256;   // threads per CTA
constexpr int AS_STRIDE = BK + 4;
constexpr int MAX_SLOTS = 2 * CAPE_MAX_TERMS;

struct TermDev {
  const float* src;
  OpView op;
  int F, src_rows, src_stride, w_stride, w2_stride;
  const float* w;
  const float* w2;
  const float* wT;    // K-major copy of w: element (f, c) = wT[c * wT_stride + f] (tensor-core path), or nullptr
  const float* w2T;
  int wT_stride, w2T_stride;
  int vec;
  const float* wT_lo;   // optional: wT - trunc_tf32(wT), same layout (not read by the wgmma kernels)
  const float* w2T_lo;
  float* stash;       // optional copy of the gathered basis rows [total_rows, stash_stride] (cape_term.stash)
  int stash_stride;
};

struct ConvParams {
  int N, rows_out, ncols, nterms;
  long long total_rows;
  TermDev terms[CAPE_MAX_TERMS];
  // condition slots: (term, accumulator) pairs that carry condition weights
  int nslots;
  int slot_term[MAX_SLOTS];
  int slot_acc[MAX_SLOTS];
  const float* slot_w[MAX_SLOTS];
  const float* cond;
  int C;
  int epilogue, act;
  float alpha;
  const float* bias;
  int bias_per_row;
  // terms[0, nterms) are contracted; terms[nterms, nterms + npass) are pass-through terms (cape_term with no weights:
  // acc0 += op . src[:, :, :ncols] in the epilogue).  A launcher that does not add them must decline a call with npass > 0.
  // (Here it fills the padding before `aux`: the layout of the other fields is unchanged.)
  int npass;
  const float* aux;
  float* out;
  float* out2;
  int wvec, ovec;
};

// One row of a pass-through term: sum_j op[r, j] * base[idx[r, j] * stride] (op.idx == nullptr: base[r * stride]), taps in
// table order.  `base` points at the sample's source rows, offset by the column.
__device__ __forceinline__ float pass_row(const OpView& op, int r, const float* base, size_t stride) {
  if (op.idx == nullptr) return __ldg(base + (size_t)r * stride);
  const int32_t* ip = op.idx + (size_t)r * op.width;
  const float* wp = op.w + (size_t)r * op.width;
  float v = 0.f;
  for (int j = 0; j < op.width; ++j) {
    const int id = __ldg(ip + j);
    if (id < 0) break;
    v = fmaf(__ldg(wp + j), __ldg(base + (size_t)id * stride), v);
  }
  return v;
}

// the same for two adjacent columns (base 8-byte aligned, stride even)
__device__ __forceinline__ float2 pass_row2(const OpView& op, int r, const float* base, size_t stride) {
  if (op.idx == nullptr) return __ldg(reinterpret_cast<const float2*>(base + (size_t)r * stride));
  const int32_t* ip = op.idx + (size_t)r * op.width;
  const float* wp = op.w + (size_t)r * op.width;
  float2 v = make_float2(0.f, 0.f);
  for (int j = 0; j < op.width; ++j) {
    const int id = __ldg(ip + j);
    if (id < 0) break;
    const float w = __ldg(wp + j);
    const float2 s = __ldg(reinterpret_cast<const float2*>(base + (size_t)id * stride));
    v.x = fmaf(w, s.x, v.x);
    v.y = fmaf(w, s.y, v.y);
  }
  return v;
}

// all-plain-operand calls (every term an identity operator) on the wgmma kernel (ellconv_tc.cu): 1 = launched, 0 = not eligible
int launch_gemm_tc(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st);
// wgmma path (ellconv_tc.cu): returns 1 if it launched, 0 if the problem is not eligible, <0 on error.
int launch_ellconv_tc(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st);
bool tensor_cores_enabled();
// thin-input layers (thin.cu): sources with <= 4 channels.  1 = launched, 0 = not eligible, <0 = error
int launch_thin_fwd(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st);
// thin-output layers (<= 4 columns): project, then combine
int launch_thinout_fwd(const cape_topology* t, const ConvParams& p, bool dual, cudaStream_t st);
int launch_thin_dw(const cape_topology* t, const cape_dw_args* a, const OpView* ops, int nops, int* nsplit_out,
                   cudaStream_t st);
// wgmma weight-gradient path (ellconv_dw_tc.cu), plain or gathered basis: 1 = launched (partials in the workspace if *nsplit_out > 1)
int launch_ellconv_dw_tc(const cape_topology* t, const cape_dw_args* a, const OpView& op, int* nsplit_out,
                         cudaStream_t st);

// experiment knobs (cape_set_tuning): [7] = 1: thin-output layers on the generic kernels, [8] = 1: no tensor-core
// plain-operand path, [10]: rows per cape_apply CTA, [16] = 1: scalar FC kernel, [17] = 1: fixed thin-dW CTA count
extern int g_tuning[32];

}  // namespace cape
