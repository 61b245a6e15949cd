// TensorBoard summaries on the device: per-variable weight histograms (tf.summary.histogram of every graph-conv weight
// and bias, lib/models.py:217-227) and the moving averages of the two loss totals (lib/models.py:393-414).
#include <climits>
#include <cmath>

#include "common.cuh"

namespace cape {

constexpr int HIST_THREADS = 256;
constexpr int HIST_WARPS = HIST_THREADS / 32;
// blocks per segment: block j of a segment takes the j-th contiguous slice of it, so the partials, and with them the
// double sums, are combined in one fixed order
constexpr int HIST_SLICES = 32;
constexpr int HIST_MAX_LIMITS = 3072;   // limits (double) + counts (u32) in shared memory: 36 KB at most

// what one block found in its slice (finite values only); min / max carry the index of their first occurrence, so that
// a -0.0 / +0.0 tie resolves as TF's sequential `if (value < min_)` does: the earlier element wins
struct HistPartial {
  double sum, sumsq;
  long long num, nonfinite, mn_i, mx_i;
  float mn, mx;
};

__device__ __forceinline__ void take_min(float& v, long long& i, float v2, long long i2) {
  if (v2 < v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}
__device__ __forceinline__ void take_max(float& v, long long& i, float v2, long long i2) {
  if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}

__device__ __forceinline__ void warp_combine(HistPartial& p) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    p.sum += __shfl_down_sync(0xffffffffu, p.sum, o);
    p.sumsq += __shfl_down_sync(0xffffffffu, p.sumsq, o);
    p.num += __shfl_down_sync(0xffffffffu, p.num, o);
    p.nonfinite += __shfl_down_sync(0xffffffffu, p.nonfinite, o);
    const float mn = __shfl_down_sync(0xffffffffu, p.mn, o), mx = __shfl_down_sync(0xffffffffu, p.mx, o);
    const long long mn_i = __shfl_down_sync(0xffffffffu, p.mn_i, o), mx_i = __shfl_down_sync(0xffffffffu, p.mx_i, o);
    take_min(p.mn, p.mn_i, mn, mn_i);
    take_max(p.mx, p.mx_i, mx, mx_i);
  }
}

__device__ __forceinline__ void combine(HistPartial& a, const HistPartial& b) {
  a.sum += b.sum;
  a.sumsq += b.sumsq;
  a.num += b.num;
  a.nonfinite += b.nonfinite;
  take_min(a.mn, a.mn_i, b.mn, b.mn_i);
  take_max(a.mx, a.mx_i, b.mx, b.mx_i);
}

// grid (HIST_SLICES, nseg).  counts and arrivals are zero on entry; the last block of a segment to finish adds the
// HIST_SLICES partials up in slice order and writes the segment's stats.
__global__ void __launch_bounds__(HIST_THREADS) histogram_kernel(const cape_hist_segment* __restrict__ segs,
                                                                 const double* __restrict__ limits, int nlim,
                                                                 double* __restrict__ stats,
                                                                 int64_t* __restrict__ nonfinite,
                                                                 unsigned long long* __restrict__ counts,
                                                                 HistPartial* __restrict__ partials,
                                                                 unsigned int* __restrict__ arrivals) {
  extern __shared__ double smem[];
  double* lim = smem;
  unsigned int* cnt = reinterpret_cast<unsigned int*>(smem + nlim);
  __shared__ HistPartial wred[HIST_WARPS];
  __shared__ bool last;
  const int s = blockIdx.y, j = blockIdx.x;
  for (int i = threadIdx.x; i < nlim; i += HIST_THREADS) {
    lim[i] = limits[i];
    cnt[i] = 0u;
  }
  __syncthreads();
  const cape_hist_segment sg = segs[s];
  const long long per = (sg.n + HIST_SLICES - 1) / HIST_SLICES;
  const long long lo = j * per, hi = min((long long)sg.n, lo + per);
  HistPartial p;
  p.sum = 0.0; p.sumsq = 0.0; p.num = 0; p.nonfinite = 0;
  p.mn = INFINITY; p.mx = -INFINITY; p.mn_i = LLONG_MAX; p.mx_i = LLONG_MAX;
  for (long long i = lo + threadIdx.x; i < hi; i += HIST_THREADS) {
    const float x = __ldg(sg.p + i);
    if (!isfinite(x)) {
      ++p.nonfinite;
      continue;
    }
    // std::upper_bound in double: the first limit greater than x (the last limit is DBL_MAX, so it exists)
    const double d = (double)x;
    int a = 0, b = nlim;
    while (a < b) {
      const int m = (a + b) >> 1;
      if (lim[m] <= d) a = m + 1;
      else b = m;
    }
    atomicAdd(cnt + a, 1u);
    take_min(p.mn, p.mn_i, x, i);
    take_max(p.mx, p.mx_i, x, i);
    ++p.num;
    p.sum += d;
    p.sumsq += d * d;
  }
  warp_combine(p);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) wred[wid] = p;
  __syncthreads();
  for (int i = threadIdx.x; i < nlim; i += HIST_THREADS)
    if (cnt[i]) atomicAdd(counts + (size_t)s * nlim + i, (unsigned long long)cnt[i]);
  if (threadIdx.x == 0) {
    HistPartial t = wred[0];
    for (int w = 1; w < HIST_WARPS; ++w) combine(t, wred[w]);
    partials[(size_t)s * HIST_SLICES + j] = t;
    __threadfence();
    last = atomicAdd(arrivals + s, 1u) == HIST_SLICES - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  const volatile HistPartial* vp = partials + (size_t)s * HIST_SLICES;
  HistPartial t;
  t.sum = vp[0].sum; t.sumsq = vp[0].sumsq; t.num = vp[0].num; t.nonfinite = vp[0].nonfinite;
  t.mn = vp[0].mn; t.mx = vp[0].mx; t.mn_i = vp[0].mn_i; t.mx_i = vp[0].mx_i;
  for (int k = 1; k < HIST_SLICES; ++k) {
    HistPartial u;
    u.sum = vp[k].sum; u.sumsq = vp[k].sumsq; u.num = vp[k].num; u.nonfinite = vp[k].nonfinite;
    u.mn = vp[k].mn; u.mx = vp[k].mx; u.mn_i = vp[k].mn_i; u.mx_i = vp[k].mx_i;
    combine(t, u);
  }
  double* o = stats + (size_t)s * 5;
  // no finite value: TF's empty histogram (Histogram::Clear: min = DBL_MAX, max = -DBL_MAX)
  o[0] = t.num ? (double)t.mn : limits[nlim - 1];
  o[1] = t.num ? (double)t.mx : -limits[nlim - 1];
  o[2] = (double)t.num;
  o[3] = t.sum;
  o[4] = t.sumsq;
  nonfinite[s] = t.nonfinite;
}

// One thread: TF-1 evaluates the loss totals op by op in fp32 (no fused multiply-add), left to right, and
// ExponentialMovingAverage's assign_moving_average does  s -= (s - v) * (1 - decay)  with (1 - decay) itself an fp32 op.
__global__ void loss_ema_kernel(const float* __restrict__ losses, const float* __restrict__ fc_sumsq, float lam_gan,
                                float lam_recon, float lam_edge, float lam_latent, float reg, float decay,
                                float* __restrict__ shadow) {
  // reg_g = r * sum_W r * l2_loss(W), l2_loss(W) = sum(W^2) / 2
  const float reg_g = __fmul_rn(reg, __fmul_rn(reg, __fmul_rn(*fc_sumsq, 0.5f)));
  float g = __fmul_rn(losses[3], lam_gan);
  g = __fadd_rn(g, __fmul_rn(losses[0], lam_recon));
  g = __fadd_rn(g, 0.f);
  g = __fadd_rn(g, __fmul_rn(losses[1], lam_edge));
  g = __fadd_rn(g, __fmul_rn(losses[2], lam_latent));
  g = __fadd_rn(g, reg_g);
  const float d = __fadd_rn(__fmul_rn(__fadd_rn(losses[4], losses[5]), lam_gan), 0.f);   // + fc_regularization_d = 0
  const float k = __fsub_rn(1.f, decay);
  shadow[0] = __fsub_rn(shadow[0], __fmul_rn(__fsub_rn(shadow[0], g), k));
  shadow[1] = __fsub_rn(shadow[1], __fmul_rn(__fsub_rn(shadow[1], d), k));
}

}  // namespace cape

using namespace cape;

extern "C" int cape_histogram(cape_topology* t, const cape_hist_segment* segs, int nseg, const double* limits, int nlim,
                              double* stats, int64_t* nonfinite, int64_t* counts, void* stream) {
  CAPE_REQUIRE(t && segs && limits && stats && nonfinite && counts, "null pointer");
  CAPE_REQUIRE(nseg > 0 && nseg <= 65535, "bad segment count");
  CAPE_REQUIRE(nlim >= 1 && nlim <= HIST_MAX_LIMITS, "bad number of bucket limits");
  const size_t part_bytes = (size_t)nseg * HIST_SLICES * sizeof(HistPartial);
  CAPE_REQUIRE((int64_t)(part_bytes + (size_t)nseg * sizeof(unsigned int)) <= t->workspace_bytes,
               "workspace too small for the histogram");
  cudaStream_t st = (cudaStream_t)stream;
  HistPartial* partials = (HistPartial*)t->workspace;
  unsigned int* arrivals = (unsigned int*)((char*)t->workspace + part_bytes);
  CAPE_CHECK_CUDA(cudaMemsetAsync(arrivals, 0, (size_t)nseg * sizeof(unsigned int), st));
  CAPE_CHECK_CUDA(cudaMemsetAsync(counts, 0, (size_t)nseg * nlim * sizeof(int64_t), st));
  const size_t shm = (size_t)nlim * (sizeof(double) + sizeof(unsigned int));
  histogram_kernel<<<dim3(HIST_SLICES, (unsigned)nseg), HIST_THREADS, shm, st>>>(
      segs, limits, nlim, stats, nonfinite, reinterpret_cast<unsigned long long*>(counts), partials, arrivals);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_loss_ema(const float* losses, const float* fc_sumsq, float lambda_gan, float lambda_recon,
                             float lambda_edge, float lambda_latent, float regularization, float decay, float* shadow,
                             void* stream) {
  CAPE_REQUIRE(losses && fc_sumsq && shadow, "null pointer");
  CAPE_REQUIRE(decay >= 0.f && decay <= 1.f, "decay must be in [0, 1]");
  loss_ema_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(losses, fc_sumsq, lambda_gan, lambda_recon, lambda_edge,
                                                     lambda_latent, regularization, decay, shadow);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}
