// Group normalisation + ReLU for the non-affine decoder residual blocks
// (CAPE.gn at lib/models.py:681-712 followed by tf.nn.relu at :752,756,760).
// Layout [N, rows, C]: the statistics of group g of sample n span (C/G contiguous channels) x (all rows),
// biased variance (tf.nn.moments), eps inside the sqrt.  Group sums are accumulated in fp64 so the
// E[x^2]-E[x]^2 form stays within fp32 rounding of the two-pass reference.
#include "common.cuh"

namespace cape {

constexpr int GN_ROWS = 64;      // rows per CTA in the reduction passes
constexpr int GN_MAXG = 32;

// Partial sums of one block of rows: thread = (row slot, float4 column); per-thread register sums over its rows, a
// shared-memory reduction over the row slots, then one fp64 atomic per group and block.
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, int rows, int C, int G,
                                                       int rows_per_block, double* __restrict__ acc) {
  __shared__ float red[2][1024];
  const int n = blockIdx.y, cpr = C >> 2, rslots = min(256 / cpr, 32);
  const int rs = threadIdx.x / cpr, c4 = threadIdx.x % cpr;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  if (rs < rslots) {
    const float4* xp = reinterpret_cast<const float4*>(x + (size_t)n * rows * C) + c4;
    for (int r = r0 + rs; r < r1; r += rslots) {
      const float4 v = __ldg(xp + (size_t)r * cpr);
      s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
      q[0] = fmaf(v.x, v.x, q[0]); q[1] = fmaf(v.y, v.y, q[1]); q[2] = fmaf(v.z, v.z, q[2]); q[3] = fmaf(v.w, v.w, q[3]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { red[0][rs * C + c4 * 4 + j] = s[j]; red[1][rs * C + c4 * 4 + j] = q[j]; }
  }
  __syncthreads();
  if (threadIdx.x < G) {
    const int cpg = C / G;
    double ds = 0.0, dq = 0.0;
    for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c)
      for (int k = 0; k < rslots; ++k) { ds += (double)red[0][k * C + c]; dq += (double)red[1][k * C + c]; }
    atomicAdd(acc + ((size_t)n * G + threadIdx.x) * 2 + 0, ds);
    atomicAdd(acc + ((size_t)n * G + threadIdx.x) * 2 + 1, dq);
  }
}

__global__ void gn_finalize_kernel(const double* __restrict__ acc, int total, double inv_cnt, float eps,
                                   float* __restrict__ stats) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const double mean = acc[2 * i] * inv_cnt;
  double var = acc[2 * i + 1] * inv_cnt - mean * mean;
  if (var < 0.0) var = 0.0;
  stats[2 * i] = (float)mean;
  stats[2 * i + 1] = (float)(1.0 / sqrt(var + (double)eps));
}

// y = relu(gamma * (x - mean) * rstd + beta): blockIdx.y = sample, float4 per thread, 32-bit index arithmetic
__global__ void __launch_bounds__(256) gn_apply_kernel(const float* __restrict__ x, int rows, int C, int G,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       const float* __restrict__ stats, float* __restrict__ y) {
  const int n = blockIdx.y, cpg = C / G, c4n = C >> 2;
  const unsigned per = (unsigned)rows * (unsigned)c4n;
  const float4* xp = reinterpret_cast<const float4*>(x + (size_t)n * rows * C);
  float4* yp = reinterpret_cast<float4*>(y + (size_t)n * rows * C);
  const float* st = stats + (size_t)n * G * 2;
  for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < per; e += gridDim.x * blockDim.x) {
    const int c = (int)(e % (unsigned)c4n) * 4;
    const float4 v = __ldg(xp + e);
    const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + c)), bt = __ldg(reinterpret_cast<const float4*>(beta + c));
    const float in[4] = {v.x, v.y, v.z, v.w}, g4[4] = {gm.x, gm.y, gm.z, gm.w}, b4[4] = {bt.x, bt.y, bt.z, bt.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* sg = st + ((c + j) / cpg) * 2;
      o[j] = fmaxf((in[j] - sg[0]) * sg[1] * g4[j] + b4[j], 0.f);
    }
    yp[e] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// pass 1 of backward: per-channel sums (dgamma, dbeta) and per-(n,g) sums of dxhat and dxhat*xhat
__global__ void __launch_bounds__(256) gn_bwd_stats_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                           const float* __restrict__ dy, int rows, int C, int G,
                                                           int rows_per_block, const float* __restrict__ gamma,
                                                           const float* __restrict__ stats, float* __restrict__ dgamma,
                                                           float* __restrict__ dbeta, double* __restrict__ acc) {
  __shared__ float red[2][1024];
  const int n = blockIdx.y, cpr = C >> 2, rslots = min(256 / cpr, 32), cpg = C / G;
  const int rs = threadIdx.x / cpr, c4 = threadIdx.x % cpr;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  if (rs < rslots) {
    float mean[4], rstd[4], sb[4] = {0.f, 0.f, 0.f, 0.f}, sg[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t g = (size_t)n * G + (c4 * 4 + j) / cpg;
      mean[j] = stats[g * 2]; rstd[j] = stats[g * 2 + 1];
    }
    const size_t base = (size_t)n * rows * C;
    const float4* xp = reinterpret_cast<const float4*>(x + base) + c4;
    const float4* yp = reinterpret_cast<const float4*>(y + base) + c4;
    const float4* dp = reinterpret_cast<const float4*>(dy + base) + c4;
    for (int r = r0 + rs; r < r1; r += rslots) {
      const float4 xv = __ldg(xp + (size_t)r * cpr), yv = __ldg(yp + (size_t)r * cpr), dv = __ldg(dp + (size_t)r * cpr);
      const float xi[4] = {xv.x, xv.y, xv.z, xv.w}, yi[4] = {yv.x, yv.y, yv.z, yv.w}, di[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float gy = (yi[j] > 0.f) ? di[j] : 0.f;
        sb[j] += gy;
        sg[j] = fmaf(gy, (xi[j] - mean[j]) * rstd[j], sg[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { red[0][rs * C + c4 * 4 + j] = sb[j]; red[1][rs * C + c4 * 4 + j] = sg[j]; }
  }
  __syncthreads();
  // per-channel totals of the block: dbeta / dgamma, and (kept in red[.][c]) the inputs of the group sums
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float b = 0.f, g = 0.f;
    for (int k = 0; k < rslots; ++k) { b += red[0][k * C + c]; g += red[1][k * C + c]; }
    atomicAdd(dbeta + c, b);
    atomicAdd(dgamma + c, g);
    const float gm = __ldg(gamma + c);
    red[0][c] = gm * b; red[1][c] = gm * g;            // slot k = 0 is only read by this thread above
  }
  __syncthreads();
  if (threadIdx.x < G) {
    double d0 = 0.0, d1 = 0.0;
    for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; ++c) { d0 += (double)red[0][c]; d1 += (double)red[1][c]; }
    atomicAdd(acc + ((size_t)n * G + threadIdx.x) * 2 + 0, d0);
    atomicAdd(acc + ((size_t)n * G + threadIdx.x) * 2 + 1, d1);
  }
}

__global__ void __launch_bounds__(256) gn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                           const float* __restrict__ dy, int rows, int C, int G,
                                                           const float* __restrict__ gamma, const float* __restrict__ stats,
                                                           const double* __restrict__ acc, double inv_cnt,
                                                           float* __restrict__ dx, int accumulate) {
  const int n = blockIdx.y, cpg = C / G, c4n = C >> 2;
  const unsigned per = (unsigned)rows * (unsigned)c4n;
  const size_t base = (size_t)n * rows * C;
  const float4* xp = reinterpret_cast<const float4*>(x + base);
  const float4* yp = reinterpret_cast<const float4*>(y + base);
  const float4* dyp = reinterpret_cast<const float4*>(dy + base);
  float4* dxp = reinterpret_cast<float4*>(dx + base);
  for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < per; e += gridDim.x * blockDim.x) {
    const int c = (int)(e % (unsigned)c4n) * 4;
    const float4 xv = __ldg(xp + e), yv = __ldg(yp + e), dv = __ldg(dyp + e);
    const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + c));
    const float xi[4] = {xv.x, xv.y, xv.z, xv.w}, yi[4] = {yv.x, yv.y, yv.z, yv.w}, di[4] = {dv.x, dv.y, dv.z, dv.w};
    const float g4[4] = {gm.x, gm.y, gm.z, gm.w};
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const size_t sg = (size_t)n * G + (c + j) / cpg;
      const float mean = stats[sg * 2], rstd = stats[sg * 2 + 1];
      const float m1 = (float)(acc[sg * 2] * inv_cnt), m2 = (float)(acc[sg * 2 + 1] * inv_cnt);
      const float gy = (yi[j] > 0.f) ? di[j] : 0.f;
      const float xh = (xi[j] - mean) * rstd;
      o[j] = rstd * (g4[j] * gy - m1 - xh * m2);
    }
    if (accumulate) {
      const float4 p = dxp[e];
      o[0] += p.x; o[1] += p.y; o[2] += p.z; o[3] += p.w;
    }
    dxp[e] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace cape

using namespace cape;

static int gn_check(cape_topology* t, int N, int rows, int C, int G) {
  CAPE_REQUIRE(t, "null handle");
  CAPE_REQUIRE(N > 0 && rows > 0 && C > 0 && G > 0 && G <= GN_MAXG && C % G == 0, "bad group-norm shape");
  CAPE_REQUIRE(C % 4 == 0 && C <= 1024, "group norm needs C % 4 == 0 (float4 rows) and C <= 1024");
  CAPE_REQUIRE((int64_t)N * G * 2 * (int64_t)sizeof(double) <= t->workspace_bytes, "workspace too small for group norm");
  CAPE_REQUIRE(N <= 65535, "batch too large");
  return 0;
}

extern "C" int cape_gn_relu_fwd(cape_topology* t, const float* x, int N, int rows, int C, int G, float eps,
                                const float* gamma, const float* beta, float* y, float* stats, void* stream) {
  if (gn_check(t, N, rows, C, G) != 0) return -1;
  CAPE_REQUIRE(x && gamma && beta && y && stats, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  double* acc = (double*)t->workspace;
  CAPE_CHECK_CUDA(cudaMemsetAsync(acc, 0, (size_t)N * G * 2 * sizeof(double), st));
  dim3 grid((rows + GN_ROWS - 1) / GN_ROWS, N);
  gn_stats_kernel<<<grid, 256, 0, st>>>(x, rows, C, G, GN_ROWS, acc);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  const double inv_cnt = 1.0 / ((double)rows * (C / G));
  gn_finalize_kernel<<<(N * G + 127) / 128, 128, 0, st>>>(acc, N * G, inv_cnt, eps, stats);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  {
    long long bx = ((long long)rows * (C / 4) + 255) / 256;
    const long long cap = ((long long)H100_SMS * 16 + N - 1) / N;
    if (bx > cap) bx = cap;
    gn_apply_kernel<<<dim3((unsigned)bx, (unsigned)N), 256, 0, st>>>(x, rows, C, G, gamma, beta, stats, y);
  }
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_gn_relu_bwd(cape_topology* t, const float* x, const float* y, const float* dy, int N, int rows,
                                int C, int G, const float* gamma, const float* stats, float* dx, int accumulate_dx,
                                float* dgamma, float* dbeta, void* stream) {
  if (gn_check(t, N, rows, C, G) != 0) return -1;
  CAPE_REQUIRE(x && y && dy && gamma && stats && dx && dgamma && dbeta, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  double* acc = (double*)t->workspace;
  CAPE_CHECK_CUDA(cudaMemsetAsync(acc, 0, (size_t)N * G * 2 * sizeof(double), st));
  dim3 grid((rows + GN_ROWS - 1) / GN_ROWS, N);
  gn_bwd_stats_kernel<<<grid, 256, 0, st>>>(x, y, dy, rows, C, G, GN_ROWS, gamma, stats, dgamma, dbeta, acc);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  const double inv_cnt = 1.0 / ((double)rows * (C / G));
  {
    long long bx = ((long long)rows * (C / 4) + 255) / 256;
    const long long cap = ((long long)H100_SMS * 16 + N - 1) / N;
    if (bx > cap) bx = cap;
    gn_bwd_apply_kernel<<<dim3((unsigned)bx, (unsigned)N), 256, 0, st>>>(x, y, dy, rows, C, G, gamma, stats, acc, inv_cnt, dx,
                                                                         accumulate_dx);
  }
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}
