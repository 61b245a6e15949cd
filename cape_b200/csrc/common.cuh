// Internal helpers shared by the kernels of libcape_b200.so (not part of the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "../../include/cape_b200.h"

namespace cape {

// SM count of the H100 SXM: grid caps of the grid-stride kernels are small multiples of it
constexpr int H100_SMS = 132;

void set_error(const std::string& msg);
void count_launches(int n);   // bookkeeping for cape_launch_count()

#define CAPE_CHECK_CUDA(expr)                                                              \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      cape::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                 \
      return -2;                                                                           \
    }                                                                                      \
  } while (0)

#define CAPE_REQUIRE(cond, msg)                                                            \
  do {                                                                                     \
    if (!(cond)) {                                                                         \
      cape::set_error(std::string("invalid argument: ") + (msg));                          \
      return -1;                                                                           \
    }                                                                                      \
  } while (0)

struct EllOp {
  int rows_out = 0, rows_in = 0, width = 0;
  int32_t* idx = nullptr;   // device [rows_out, width], -1 = empty slot
  float* w = nullptr;       // device [rows_out, width]
  float* rowsum = nullptr;  // device [rows_out]
};

}  // namespace cape

struct cape_topology {
  int device = 0;
  int sm_count = cape::H100_SMS;   // replaced by the device's count when the handle is created
  std::vector<cape::EllOp> ops;
  void* workspace = nullptr;
  int64_t workspace_bytes = 0;
  // tile ticket of the persistent conv_wg_kernel (ellconv_tc.cu): device int, zero between launches.  Every launch
  // that uses it must be ordered after the previous one (one stream, or a graph replayed on one stream).
  unsigned* tile_counter = nullptr;
};

namespace cape {

// device-side view of an operator (identity when idx == nullptr)
struct OpView {
  const int32_t* idx;
  const float* w;
  const float* rowsum;
  int width;
};

inline int get_op(const cape_topology* t, int op, int rows_out, int rows_in, OpView* v) {
  if (op < 0) {
    if (rows_in != rows_out) {
      set_error("identity operator needs src_rows == rows_out");
      return -1;
    }
    v->idx = nullptr; v->w = nullptr; v->rowsum = nullptr; v->width = 0;
    return 0;
  }
  if (op >= (int)t->ops.size()) { set_error("operator id out of range"); return -1; }
  const EllOp& o = t->ops[op];
  if (o.rows_out != rows_out || o.rows_in != rows_in) {
    set_error("operator shape mismatch: op is [" + std::to_string(o.rows_out) + "x" + std::to_string(o.rows_in) +
              "], call wants [" + std::to_string(rows_out) + "x" + std::to_string(rows_in) + "]");
    return -1;
  }
  v->idx = o.idx; v->w = o.w; v->rowsum = o.rowsum; v->width = o.width;
  return 0;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void fma4(float4& a, float s, const float4& x) {
  a.x = fmaf(s, x.x, a.x); a.y = fmaf(s, x.y, a.y); a.z = fmaf(s, x.z, a.z); a.w = fmaf(s, x.w, a.w);
}

// sum_j w[r, j] * base[idx[r, j] * stride], tap by tap in table order: one scalar column
__device__ __forceinline__ float ell_gather1(const OpView& op, int r, const float* base, size_t stride) {
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

// v += sum_j w[r, j] * src_row(idx[r, j])  for one float4 column group.  Taps are fetched four at a time (the
// tables are padded to a multiple of 4, empty slots idx = -1 / w = 0) so that four independent neighbour-row loads
// are in flight per batch instead of one dependent load per tap.
__device__ __forceinline__ void ell_gather4(const OpView& op, int r, const float* base, size_t stride, float4& v) {
  const int4* ip = reinterpret_cast<const int4*>(op.idx + (size_t)r * op.width);
  const float4* wp = reinterpret_cast<const float4*>(op.w + (size_t)r * op.width);
  const int nb = op.width >> 2;
  int4 id = __ldg(ip);
  for (int b = 0; b < nb; ++b) {
    if (id.x < 0) break;
    const float4 ww = __ldg(wp + b);
    int4 idn = make_int4(-1, -1, -1, -1);
    if (b + 1 < nb) idn = __ldg(ip + b + 1);
    const float4 x0 = ldg4(base + (size_t)id.x * stride);
    const float4 x1 = ldg4(base + (size_t)max(id.y, 0) * stride);
    const float4 x2 = ldg4(base + (size_t)max(id.z, 0) * stride);
    const float4 x3 = ldg4(base + (size_t)max(id.w, 0) * stride);
    fma4(v, ww.x, x0); fma4(v, ww.y, x1); fma4(v, ww.z, x2); fma4(v, ww.w, x3);
    id = idn;
  }
}

// Two rows at once: eight independent neighbour-row loads in flight per thread (the gather is latency-bound on L2).
__device__ __forceinline__ void ell_gather4_pair(const OpView& op, int ra, int rb, const float* base_a,
                                                 const float* base_b, size_t stride, float4& va, float4& vb) {
  const int4* ipa = reinterpret_cast<const int4*>(op.idx + (size_t)ra * op.width);
  const int4* ipb = reinterpret_cast<const int4*>(op.idx + (size_t)rb * op.width);
  const float4* wpa = reinterpret_cast<const float4*>(op.w + (size_t)ra * op.width);
  const float4* wpb = reinterpret_cast<const float4*>(op.w + (size_t)rb * op.width);
  const int nb = op.width >> 2;
  int4 ia = __ldg(ipa), ib = __ldg(ipb);
  for (int b = 0; b < nb; ++b) {
    const bool da = ia.x >= 0, db = ib.x >= 0;
    if (!da && !db) break;
    // w of an exhausted row is irrelevant: its loads are redirected to row 0 and multiplied by 0
    float4 wa = make_float4(0.f, 0.f, 0.f, 0.f), wb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (da) wa = __ldg(wpa + b);
    if (db) wb = __ldg(wpb + b);
    int4 na = make_int4(-1, -1, -1, -1), nbx = make_int4(-1, -1, -1, -1);
    if (b + 1 < nb) { na = __ldg(ipa + b + 1); nbx = __ldg(ipb + b + 1); }
    const float4 a0 = ldg4(base_a + (size_t)max(ia.x, 0) * stride), a1 = ldg4(base_a + (size_t)max(ia.y, 0) * stride);
    const float4 a2 = ldg4(base_a + (size_t)max(ia.z, 0) * stride), a3 = ldg4(base_a + (size_t)max(ia.w, 0) * stride);
    const float4 b0 = ldg4(base_b + (size_t)max(ib.x, 0) * stride), b1 = ldg4(base_b + (size_t)max(ib.y, 0) * stride);
    const float4 b2 = ldg4(base_b + (size_t)max(ib.z, 0) * stride), b3 = ldg4(base_b + (size_t)max(ib.w, 0) * stride);
    fma4(va, wa.x, a0); fma4(va, wa.y, a1); fma4(va, wa.z, a2); fma4(va, wa.w, a3);
    fma4(vb, wb.x, b0); fma4(vb, wb.y, b1); fma4(vb, wb.z, b2); fma4(vb, wb.w, b3);
    ia = na; ib = nbx;
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace cape
