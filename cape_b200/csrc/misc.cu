// Small fused kernels around the graph convolutions: re-parameterisation, losses, optimiser.
// Reference: lib/models.py:193-196 (vae_sampling), :354-416 + lib/losses.py:9-25 (losses),
// :419-474 (clip_by_global_norm + MomentumOptimizer).
#include <cmath>

#include "common.cuh"

namespace cape {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum; result valid in thread 0
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float s = 0.f;
  if (wid == 0) {
    s = (lane < (int)(blockDim.x >> 5)) ? red[lane] : 0.f;
    s = warp_sum(s);
  }
  __syncthreads();
  return s;
}

__global__ void act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ g,
                               long long n, float alpha) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    g[i] = dy[i] * (y[i] > 0.f ? 1.f : alpha);
}

__global__ void axpy_kernel(float* __restrict__ y, const float* __restrict__ x, float a, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = fmaf(a, x[i], y[i]);
}

__global__ void vae_fwd_kernel(const float* __restrict__ mean, const float* __restrict__ logvar,
                               const float* __restrict__ eps, float* __restrict__ z, int z_stride, int N, int nz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * nz) return;
  const int n = i / nz, j = i % nz;
  z[(size_t)n * z_stride + j] = mean[i] + sqrtf(expf(logvar[i])) * eps[i];
}

__global__ void vae_bwd_kernel(const float* __restrict__ dz, int dz_stride, const float* __restrict__ mean,
                               const float* __restrict__ logvar, const float* __restrict__ eps,
                               float* __restrict__ dmean, float* __restrict__ dlogvar, int N, int nz, float kl_scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * nz) return;
  const int n = i / nz, j = i % nz;
  const float d = dz[(size_t)n * dz_stride + j];
  const float e = expf(logvar[i]);
  const float invN = 1.f / (float)N;
  dmean[i] = d + kl_scale * mean[i] * invN;
  dlogvar[i] = d * eps[i] * 0.5f * sqrtf(e) + kl_scale * 0.5f * (e - 1.f) * invN;
}

struct ReconParams {
  const int32_t* nbr;   // [rows, width] neighbour table (-1 padded)
  int width;
  const float* pred;
  const float* gt;
  int N, rows;
  float g_l1;     // lambda_recon / (N*rows*3)
  float delta;    // Huber threshold
  float g_edge;   // lambda_edge / (N*n_edges)
  float s_l1;     // 1 / (N*rows*3)
  float s_edge;   // 0.5 / (N*n_edges)   (every undirected edge is visited from both ends)
  float* dpred;
  float* losses;
  const float* vweight;  // [rows] per-vertex weights of the reconstruction term (WEIGHTED instantiations only)
};

// the reconstruction term's value and gradient (before the lambda / count scale) of one coordinate's residual d
template <int KIND>
__device__ __forceinline__ float recon_term(float d, float delta, float* grad) {
  if (KIND == CAPE_RECON_L2) {
    *grad = 2.f * d;
    return d * d;
  }
  const float a = fabsf(d);
  if (KIND == CAPE_RECON_HUBER) {
    const float q = fminf(a, delta);
    *grad = fminf(fmaxf(d, -delta), delta);
    return 0.5f * q * q + delta * (a - q);
  }
  *grad = (float)((d > 0.f) - (d < 0.f));
  return a;
}

// WEIGHTED: the reconstruction term of vertex v (its three coordinates' loss and gradient) is scaled by vweight[v], and
// g_l1 / s_l1 divide by N * 3 * sum(vweight) instead of the coordinate count.  A template flag, so that the unweighted
// instantiations compile to the code they had before the flag existed.
template <int KIND, bool WEIGHTED>
__global__ void __launch_bounds__(256) recon_kernel(const __grid_constant__ ReconParams p) {
  __shared__ float red[8];
  const long long total = (long long)p.N * p.rows;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float l1 = 0.f, le = 0.f;
  if (i < total) {
    const int n = (int)(i / p.rows), v = (int)(i % p.rows);
    const float* pp = p.pred + (size_t)n * p.rows * 3;
    const float* gg = p.gt + (size_t)n * p.rows * 3;
    const float dx = pp[v * 3] - gg[v * 3], dy = pp[v * 3 + 1] - gg[v * 3 + 1], dz = pp[v * 3 + 2] - gg[v * 3 + 2];
    float tx, ty, tz;
    const float vx = recon_term<KIND>(dx, p.delta, &tx), vy = recon_term<KIND>(dy, p.delta, &ty),
                vz = recon_term<KIND>(dz, p.delta, &tz);
    l1 = vx + vy + vz;
    float g_l1 = p.g_l1;
    if (WEIGHTED) {
      const float m = __ldg(p.vweight + v);
      l1 *= m;
      g_l1 *= m;
    }
    float gx = g_l1 * tx;
    float gy = g_l1 * ty;
    float gz = g_l1 * tz;
    const int32_t* nb = p.nbr + (size_t)v * p.width;
    for (int j = 0; j < p.width; ++j) {
      const int u = __ldg(nb + j);
      if (u < 0) break;
      const float ex = dx - (pp[u * 3] - gg[u * 3]);
      const float ey = dy - (pp[u * 3 + 1] - gg[u * 3 + 1]);
      const float ez = dz - (pp[u * 3 + 2] - gg[u * 3 + 2]);
      const float len = sqrtf(ex * ex + ey * ey + ez * ez);
      le += len;
      if (len > 0.f) {
        const float s = p.g_edge / len;
        gx = fmaf(s, ex, gx); gy = fmaf(s, ey, gy); gz = fmaf(s, ez, gz);
      }
    }
    float* dp = p.dpred + (size_t)i * 3;
    dp[0] += gx; dp[1] += gy; dp[2] += gz;
  }
  const float s1 = block_sum(l1 * p.s_l1, red);
  const float s2 = block_sum(le * p.s_edge, red);
  if (threadIdx.x == 0) {
    atomicAdd(p.losses + 0, s1);
    atomicAdd(p.losses + 1, s2);
  }
}

__global__ void kl_kernel(const float* __restrict__ mean, const float* __restrict__ logvar, int total, float invN,
                          float* losses) {
  __shared__ float red[8];
  float s = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const float m = mean[i], lv = logvar[i];
    s += -0.5f * (1.f + lv - m * m - expf(lv));
  }
  const float tot = block_sum(s * invN, red);
  if (threadIdx.x == 0) atomicAdd(losses + 2, tot);
}

__global__ void bce_kernel(const float* __restrict__ logits, long long n, float label, float gscale, float lscale,
                           float* __restrict__ dlogits, float* loss) {
  __shared__ float red[8];
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float l = logits[i];
    s += fmaxf(l, 0.f) - l * label + log1pf(expf(-fabsf(l)));
    if (dlogits) {
      const float sig = 1.f / (1.f + expf(-l));
      dlogits[i] = (sig - label) * gscale;
    }
  }
  const float tot = block_sum(s * lscale, red);
  if (threadIdx.x == 0 && loss) atomicAdd(loss, tot);
}

// Deterministic: block partial sums go to a scratch array and the LAST block to finish adds them up in index order, so
// the global norm (and with it the clip factor of the update) is bit-identical on every data-parallel replica and in
// every run -- a float atomicAdd per block is not, and replicas that clip would drift apart by an ulp per step.
constexpr int SUMSQ_MAX_BLOCKS = H100_SMS * 4;
__device__ float g_sumsq_partials[SUMSQ_MAX_BLOCKS];
__device__ unsigned int g_sumsq_counter = 0;

__global__ void sumsq_kernel(const float* __restrict__ g, long long n, float* out) {
  float* partials = g_sumsq_partials;
  unsigned int* counter = &g_sumsq_counter;
  __shared__ float red[8];
  __shared__ bool last;
  float s = 0.f;
  const long long n4 = n / 4;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = g4[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    s += g[i] * g[i];
  const float tot = block_sum(s, red);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = tot;
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  float t = 0.f;
  for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) t += __ldcg(partials + i);
  const float all = block_sum(t, red);
  if (threadIdx.x == 0) {
    *out += all;
    *counter = 0;
  }
}

__global__ void sgd_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ mom, long long n,
                           const float* __restrict__ sumsq, float clip, const float* __restrict__ lr_dev,
                           float momentum) {
  float coef = 1.f;
  if (sumsq) {
    const float norm = sqrtf(*sumsq);
    coef = clip / fmaxf(norm, clip);
  }
  const float lr = *lr_dev;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float a = fmaf(momentum, mom[i], coef * g[i]);
    mom[i] = a;
    w[i] = fmaf(-lr, a, w[i]);
  }
}

// tf.train.AdamOptimizer (lib/models.py:449-451): m = b1 m + (1 - b1) g; v = b2 v + (1 - b2) g^2;
// w -= lr_t m / (sqrt(v) + eps) with lr_t = lr sqrt(1 - b2^t) / (1 - b1^t) -- the caller puts lr_t in device memory
__global__ void adam_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, long long n, const float* __restrict__ sumsq, float clip,
                            const float* __restrict__ lr_dev, float beta1, float beta2, float eps) {
  float coef = 1.f;
  if (sumsq) {
    const float norm = sqrtf(*sumsq);
    coef = clip / fmaxf(norm, clip);
  }
  const float lr = *lr_dev;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = coef * g[i];
    const float mi = fmaf(beta1, m[i], (1.f - beta1) * gi);
    const float vi = fmaf(beta2, v[i], (1.f - beta2) * gi * gi);
    m[i] = mi;
    v[i] = vi;
    w[i] -= lr * mi / (sqrtf(vi) + eps);
  }
}

__global__ void wtrans_kernel(const float* __restrict__ w, int Fin, int K, int Fout, float* __restrict__ wt) {
  // tile transpose through shared memory: for each k, [Fin x Fout] -> [Fout x Fin]
  __shared__ float tile[32][33];
  const int k = blockIdx.z;
  const int f0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int f = f0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (f < Fin && c < Fout) ? w[((size_t)f * K + k) * Fout + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, f = f0 + threadIdx.x;
    if (c < Fout && f < Fin) wt[((size_t)c * K + k) * Fin + f] = tile[threadIdx.x][i];
  }
}

// dst[i, :] = src[idx[i], :]: batch assembly from a device-resident dataset (cape_gather_rows)
__global__ void __launch_bounds__(256) gather_rows_kernel(const float* __restrict__ src, long long row_floats,
                                                          const int32_t* __restrict__ idx, int n, int n_src,
                                                          float* __restrict__ dst, int vec) {
  const int i = blockIdx.y;
  int r = __ldg(idx + i);
  r = min(max(r, 0), n_src - 1);
  const float* s = src + (size_t)r * row_floats;
  float* d = dst + (size_t)i * row_floats;
  if (vec) {
    const long long n4 = row_floats >> 2;
    for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < n4; j += (long long)gridDim.x * blockDim.x)
      reinterpret_cast<float4*>(d)[j] = __ldg(reinterpret_cast<const float4*>(s) + j);
  } else {
    for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < row_floats; j += (long long)gridDim.x * blockDim.x)
      d[j] = __ldg(s + j);
  }
}

// All derived weight layouts of many layers in one launch (cape_weight_prep): blockIdx.y = descriptor, the blocks of a
// row walk its (k, 32 x 32) tiles.  wt (k, c, f) goes through a shared-memory transpose, wk (k, f, c) is a straight copy.
__global__ void __launch_bounds__(256) wprep_kernel(const cape_wprep* __restrict__ descs) {
  __shared__ float tile[32][33];
  const cape_wprep d = descs[blockIdx.y];
  const int tf = (d.Fin + 31) / 32, tc = (d.Fout + 31) / 32;
  const int ntiles = d.K * tf * tc;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int tl = blockIdx.x; tl < ntiles; tl += gridDim.x) {
    const int k = tl / (tf * tc), f0 = ((tl / tc) % tf) * 32, c0 = (tl % tc) * 32;
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
      const int f = f0 + i, c = c0 + tx;
      const float v = (f < d.Fin && c < d.Fout) ? d.w[((size_t)f * d.K + k) * d.Fout + c] : 0.f;
      tile[i][tx] = v;
      if (d.wk != nullptr && f < d.Fin && c < d.Fout) d.wk[((size_t)k * d.Fin + f) * d.Fout + c] = v;
    }
    __syncthreads();
    if (d.wt != nullptr) {
      for (int i = ty; i < 32; i += 8) {
        const int c = c0 + i, f = f0 + tx;
        if (c < d.Fout && f < d.Fin) d.wt[((size_t)k * d.Fout + c) * d.Fin + f] = tile[tx][i];
      }
    }
  }
}

static inline int blocks_for(long long n, int threads, int cap) {
  long long b = (n + threads - 1) / threads;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace cape

using namespace cape;

extern "C" int cape_act_bwd(const float* dy, const float* y, float* g, int64_t n, float alpha, void* stream) {
  CAPE_REQUIRE(dy && y && g && n > 0, "bad arguments");
  act_bwd_kernel<<<blocks_for(n, 256, H100_SMS * 8), 256, 0, (cudaStream_t)stream>>>(dy, y, g, n, alpha);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_axpy(float* y, const float* x, float a, int64_t n, void* stream) {
  CAPE_REQUIRE(y && x && n > 0, "bad arguments");
  axpy_kernel<<<blocks_for(n, 256, H100_SMS * 8), 256, 0, (cudaStream_t)stream>>>(y, x, a, n);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_vae_sample_fwd(const float* mean, const float* logvar, const float* eps, float* z, int z_stride,
                                   int N, int nz, void* stream) {
  CAPE_REQUIRE(mean && logvar && eps && z && N > 0 && nz > 0 && z_stride >= nz, "bad arguments");
  vae_fwd_kernel<<<(N * nz + 255) / 256, 256, 0, (cudaStream_t)stream>>>(mean, logvar, eps, z, z_stride, N, nz);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_vae_sample_bwd(const float* dz, int dz_stride, const float* mean, const float* logvar,
                                   const float* eps, float* dmean, float* dlogvar, int N, int nz, float kl_scale,
                                   void* stream) {
  CAPE_REQUIRE(dz && mean && logvar && eps && dmean && dlogvar && N > 0 && nz > 0 && dz_stride >= nz, "bad arguments");
  vae_bwd_kernel<<<(N * nz + 255) / 256, 256, 0, (cudaStream_t)stream>>>(dz, dz_stride, mean, logvar, eps, dmean,
                                                                        dlogvar, N, nz, kl_scale);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

// vweight: nullptr, or [rows] per-vertex weights with their sum vweight_sum (> 0)
static int recon_losses(cape_topology* t, int nbr_op, const float* pred, const float* gt, int N, int rows, int kind,
                        float delta, float lambda_l1, float lambda_edge, int n_edges, const float* vweight,
                        double vweight_sum, const float* mean, const float* logvar, int nz, float* dpred, float* losses,
                        void* stream) {
  CAPE_REQUIRE(t && pred && gt && dpred && losses, "null pointer");
  CAPE_REQUIRE(kind == CAPE_RECON_L1 || kind == CAPE_RECON_L2 || kind == CAPE_RECON_HUBER, "unknown reconstruction loss");
  CAPE_REQUIRE(kind != CAPE_RECON_HUBER || delta > 0.f, "the Huber loss needs delta > 0");
  CAPE_REQUIRE(nbr_op >= 0 && nbr_op < (int)t->ops.size(), "bad neighbour operator");
  const EllOp& o = t->ops[nbr_op];
  CAPE_REQUIRE(o.rows_out == rows && o.rows_in == rows, "neighbour operator shape mismatch");
  CAPE_REQUIRE(N > 0 && n_edges > 0, "empty problem");
  ReconParams p{};
  p.nbr = o.idx; p.width = o.width; p.pred = pred; p.gt = gt; p.N = N; p.rows = rows;
  // TF-1 Reduction.MEAN: the weighted sum over the sum of the weights broadcast to [N, rows, 3]
  const double cnt = (double)N * (vweight ? vweight_sum : (double)rows) * 3.0, ecnt = (double)N * n_edges;
  p.g_l1 = (float)(lambda_l1 / cnt); p.g_edge = (float)(lambda_edge / ecnt);
  p.s_l1 = (float)(1.0 / cnt); p.s_edge = (float)(0.5 / ecnt);
  p.delta = delta;
  p.dpred = dpred; p.losses = losses;
  p.vweight = vweight;
  const long long total = (long long)N * rows;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (vweight) {
    if (kind == CAPE_RECON_L2) recon_kernel<CAPE_RECON_L2, true><<<blocks, 256, 0, st>>>(p);
    else if (kind == CAPE_RECON_HUBER) recon_kernel<CAPE_RECON_HUBER, true><<<blocks, 256, 0, st>>>(p);
    else recon_kernel<CAPE_RECON_L1, true><<<blocks, 256, 0, st>>>(p);
  } else {
    if (kind == CAPE_RECON_L2) recon_kernel<CAPE_RECON_L2, false><<<blocks, 256, 0, st>>>(p);
    else if (kind == CAPE_RECON_HUBER) recon_kernel<CAPE_RECON_HUBER, false><<<blocks, 256, 0, st>>>(p);
    else recon_kernel<CAPE_RECON_L1, false><<<blocks, 256, 0, st>>>(p);
  }
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  if (mean && logvar && nz > 0) {
    kl_kernel<<<blocks_for((long long)N * nz, 256, 64), 256, 0, st>>>(mean, logvar, N * nz, 1.f / (float)N, losses);
    CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  }
  return 0;
}

extern "C" int cape_recon_losses_ex(cape_topology* t, int nbr_op, const float* pred, const float* gt, int N, int rows,
                                    int kind, float delta, float lambda_l1, float lambda_edge, int n_edges,
                                    const float* mean, const float* logvar, int nz, float* dpred, float* losses,
                                    void* stream) {
  return recon_losses(t, nbr_op, pred, gt, N, rows, kind, delta, lambda_l1, lambda_edge, n_edges, nullptr, 0.0, mean,
                      logvar, nz, dpred, losses, stream);
}

extern "C" int cape_recon_losses_w(cape_topology* t, int nbr_op, const float* pred, const float* gt, int N, int rows,
                                   int kind, float delta, float lambda_l1, float lambda_edge, int n_edges,
                                   const float* vweight, double vweight_sum, const float* mean, const float* logvar,
                                   int nz, float* dpred, float* losses, void* stream) {
  CAPE_REQUIRE(vweight, "null vertex weights");
  CAPE_REQUIRE(vweight_sum > 0.0 && std::isfinite(vweight_sum), "the vertex weights must have a positive finite sum");
  return recon_losses(t, nbr_op, pred, gt, N, rows, kind, delta, lambda_l1, lambda_edge, n_edges, vweight, vweight_sum,
                      mean, logvar, nz, dpred, losses, stream);
}

extern "C" int cape_recon_losses(cape_topology* t, int nbr_op, const float* pred, const float* gt, int N, int rows,
                                 float lambda_l1, float lambda_edge, int n_edges, const float* mean,
                                 const float* logvar, int nz, float* dpred, float* losses, void* stream) {
  return cape_recon_losses_ex(t, nbr_op, pred, gt, N, rows, CAPE_RECON_L1, 0.f, lambda_l1, lambda_edge, n_edges, mean,
                              logvar, nz, dpred, losses, stream);
}

extern "C" int cape_bce_logits(const float* logits, int64_t n, float label, float scale, float* dlogits, float* loss,
                               void* stream) {
  CAPE_REQUIRE(logits && n > 0, "bad arguments");
  bce_kernel<<<blocks_for(n, 256, 256), 256, 0, (cudaStream_t)stream>>>(logits, n, label, scale / (float)n,
                                                                         1.f / (float)n, dlogits, loss);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_sumsq(const float* g, int64_t n, float* sumsq, void* stream) {
  CAPE_REQUIRE(g && sumsq && n > 0, "bad arguments");
  CAPE_REQUIRE(aligned16(g), "g must be 16-byte aligned");
  // scratch of the deterministic reduction: module-scope device variables (one copy per device, nothing to allocate, so the
  // call is capturable from the start).  Calls on one device must not overlap (same stream, or ordered).
  sumsq_kernel<<<blocks_for(n / 4 + 1, 256, SUMSQ_MAX_BLOCKS), 256, 0, (cudaStream_t)stream>>>(g, n, sumsq);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_sgd_clip_update(float* w, const float* g, float* mom, int64_t n, const float* sumsq,
                                    float clip_norm, const float* lr_dev, float momentum, void* stream) {
  CAPE_REQUIRE(w && g && mom && lr_dev && n > 0, "bad arguments");
  sgd_kernel<<<blocks_for(n, 256, H100_SMS * 8), 256, 0, (cudaStream_t)stream>>>(w, g, mom, n, sumsq, clip_norm, lr_dev,
                                                                             momentum);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_adam_clip_update(float* w, const float* g, float* m, float* v, int64_t n, const float* sumsq,
                                     float clip_norm, const float* lr_t_dev, float beta1, float beta2, float eps,
                                     void* stream) {
  CAPE_REQUIRE(w && g && m && v && lr_t_dev && n > 0, "bad arguments");
  CAPE_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && eps > 0.f, "bad Adam constants");
  adam_kernel<<<blocks_for(n, 256, H100_SMS * 8), 256, 0, (cudaStream_t)stream>>>(w, g, m, v, n, sumsq, clip_norm, lr_t_dev,
                                                                              beta1, beta2, eps);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_cheb_weight_transpose(const float* w, int Fin, int K, int Fout, float* wt, void* stream) {
  CAPE_REQUIRE(w && wt && Fin > 0 && K > 0 && Fout > 0, "bad arguments");
  dim3 grid((Fin + 31) / 32, (Fout + 31) / 32, K), block(32, 8);
  wtrans_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(w, Fin, K, Fout, wt);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_gather_rows(const float* src, int64_t row_floats, int n_src, const int32_t* idx_device, int n,
                                float* dst, void* stream) {
  CAPE_REQUIRE(src && idx_device && dst && row_floats > 0 && n > 0 && n <= 65535 && n_src > 0, "bad arguments");
  const int vec = (row_floats % 4 == 0) && aligned16(src) && aligned16(dst);
  long long per = (vec ? row_floats / 4 : row_floats);
  int bx = (int)((per + 255) / 256);
  if (bx > 32) bx = 32;
  dim3 grid((unsigned)bx, (unsigned)n);
  gather_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, row_floats, idx_device, n, n_src, dst, vec);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_weight_prep(const cape_wprep* descs_device, int n, int blocks_per_desc, void* stream) {
  CAPE_REQUIRE(descs_device && n > 0 && n <= 65535, "bad arguments");
  if (blocks_per_desc < 1) blocks_per_desc = 8;
  dim3 grid((unsigned)blocks_per_desc, (unsigned)n);
  wprep_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(descs_device);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}
