// Strided fp32 GEMM with deterministic split-K: the dense layers of CAPE
// (tf.layers.dense at lib/models.py:496,506,510,557,560,582) and their gradients.
// These are weight-bandwidth bound (2 x 55168x64 + 128x55168 fp32 = 56.7 MB read once per pass at batch 64),
// so the contraction stays on the fp32 pipe; split-K over the 55168-long reduction fills the SMs.
#include "common.cuh"
#include "ellconv_params.cuh"

namespace cape {

constexpr int G_BM = 64, G_BN = 64, G_BK = 16, G_STRIDE = 68;

struct GemmParams {
  int M, N, K;
  const float* a; long long a_rs, a_cs;
  const float* b; long long b_rs, b_cs;
  float* c; long long c_rs;
  const float* bias;
  int act;
  float leaky, alpha, beta;
  int nsplit, k_per_split;
  float* ws;
};

__device__ __forceinline__ float apply_act(float v, int act, float leaky) {
  if (act == CAPE_ACT_LEAKY) return v > 0.f ? v : leaky * v;
  if (act == CAPE_ACT_RELU) return fmaxf(v, 0.f);
  return v;
}

__device__ __forceinline__ void gemm_load(const GemmParams& p, int m0, int n0, int k0, int kend, int tid,
                                          float (&ra)[4], float (&rb)[4]) {
  if (p.a_cs == 1) {
    const int kk = tid & 15, mb = tid >> 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + mb + 16 * i, k = k0 + kk;
      ra[i] = (m < p.M && k < kend) ? __ldg(p.a + (size_t)m * p.a_rs + k) : 0.f;
    }
  } else {
    const int mm = tid & 63, kb = tid >> 6;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int m = m0 + mm, k = k0 + kb + 4 * i;
      ra[i] = (m < p.M && k < kend) ? __ldg(p.a + (size_t)m * p.a_rs + (size_t)k * p.a_cs) : 0.f;
    }
  }
  if (p.b_cs == 1) {
    const int nn = tid & 63, kb = tid >> 6;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int n = n0 + nn, k = k0 + kb + 4 * i;
      rb[i] = (n < p.N && k < kend) ? __ldg(p.b + (size_t)k * p.b_rs + n) : 0.f;
    }
  } else {
    const int kk = tid & 15, nb = tid >> 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int n = n0 + nb + 16 * i, k = k0 + kk;
      rb[i] = (n < p.N && k < kend) ? __ldg(p.b + (size_t)k * p.b_rs + (size_t)n * p.b_cs) : 0.f;
    }
  }
}

__device__ __forceinline__ void gemm_store(const GemmParams& p, int tid, const float (&ra)[4], const float (&rb)[4],
                                           float* As, float* Bs) {
  if (p.a_cs == 1) {
    const int kk = tid & 15, mb = tid >> 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) As[kk * G_STRIDE + mb + 16 * i] = ra[i];
  } else {
    const int mm = tid & 63, kb = tid >> 6;
#pragma unroll
    for (int i = 0; i < 4; ++i) As[(kb + 4 * i) * G_STRIDE + mm] = ra[i];
  }
  if (p.b_cs == 1) {
    const int nn = tid & 63, kb = tid >> 6;
#pragma unroll
    for (int i = 0; i < 4; ++i) Bs[(kb + 4 * i) * G_STRIDE + nn] = rb[i];
  } else {
    const int kk = tid & 15, nb = tid >> 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) Bs[kk * G_STRIDE + nb + 16 * i] = rb[i];
  }
}

// One 64 x 64 output tile over the reduction range [kbeg, kend).  mode 0: epilogue store (alpha, bias, act, beta),
// 1: raw partial sums to the split-K workspace slice `z`, 2: alpha * acc added atomically to c (batched accumulations).
__device__ __forceinline__ void gemm_tile(const GemmParams& p, int m0, int n0, int kbeg, int kend, int z, int mode,
                                          float* As, float* Bs) {
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  float ra[4], rb[4];
  if (kbeg < kend) gemm_load(p, m0, n0, kbeg, kend, tid, ra, rb);
  for (int k0 = kbeg; k0 < kend; k0 += G_BK) {
    gemm_store(p, tid, ra, rb, As, Bs);
    __syncthreads();
    if (k0 + G_BK < kend) gemm_load(p, m0, n0, k0 + G_BK, kend, tid, ra, rb);
#pragma unroll
    for (int kk = 0; kk < G_BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk * G_STRIDE + ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk * G_STRIDE + tx * 4]);
      acc[0][0] = fmaf(a.x, b.x, acc[0][0]); acc[0][1] = fmaf(a.x, b.y, acc[0][1]);
      acc[0][2] = fmaf(a.x, b.z, acc[0][2]); acc[0][3] = fmaf(a.x, b.w, acc[0][3]);
      acc[1][0] = fmaf(a.y, b.x, acc[1][0]); acc[1][1] = fmaf(a.y, b.y, acc[1][1]);
      acc[1][2] = fmaf(a.y, b.z, acc[1][2]); acc[1][3] = fmaf(a.y, b.w, acc[1][3]);
      acc[2][0] = fmaf(a.z, b.x, acc[2][0]); acc[2][1] = fmaf(a.z, b.y, acc[2][1]);
      acc[2][2] = fmaf(a.z, b.z, acc[2][2]); acc[2][3] = fmaf(a.z, b.w, acc[2][3]);
      acc[3][0] = fmaf(a.w, b.x, acc[3][0]); acc[3][1] = fmaf(a.w, b.y, acc[3][1]);
      acc[3][2] = fmaf(a.w, b.z, acc[3][2]); acc[3][3] = fmaf(a.w, b.w, acc[3][3]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.N) continue;
      if (mode == 1) {
        p.ws[((size_t)z * p.M + m) * p.N + n] = acc[i][j];
      } else if (mode == 2) {
        atomicAdd(p.c + (size_t)m * p.c_rs + n, p.alpha * acc[i][j]);
      } else {
        float v = p.alpha * acc[i][j];
        if (p.bias) v += __ldg(p.bias + n);
        v = apply_act(v, p.act, p.leaky);
        float* o = p.c + (size_t)m * p.c_rs + n;
        if (p.beta != 0.f) v += p.beta * (*o);
        *o = v;
      }
    }
  }
}

__global__ void __launch_bounds__(256, 2) gemm_kernel(const __grid_constant__ GemmParams p) {
  __shared__ __align__(16) float As[G_BK * G_STRIDE];
  __shared__ __align__(16) float Bs[G_BK * G_STRIDE];
  const int kbeg = blockIdx.z * p.k_per_split;
  gemm_tile(p, blockIdx.y * G_BM, blockIdx.x * G_BN, kbeg, min(p.K, kbeg + p.k_per_split), blockIdx.z,
            p.nsplit > 1 ? 1 : 0, As, Bs);
}

// ---- vectorised variant for the large skinny products (the three 28 MB FC layers and their gradients) ---------------
// The generic kernel keeps eight scalar loads per thread in flight (16 KB per SM): the FC passes ran at 0.35-0.9 TB/s.
// Here a thread prefetches two 16-byte vectors per operand for the next 64 x 64 x 32 step and three CTAs share an SM
// (48 KB in flight per SM).  AK: A is k-contiguous (a_cs == 1; else m-contiguous, a_rs == 1); BN: B is n-contiguous
// (b_cs == 1; else k-contiguous, b_rs == 1).  Eligibility (cape_gemm): every vector must be 16-byte aligned and must
// not straddle the end of its axis.
constexpr int GV_BK = 32;

template <bool AK, bool BN>
__device__ __forceinline__ void gv_load(const GemmParams& p, int m0, int n0, int k0, int kend, int tid, float4 (&ra)[2],
                                        float4 (&rb)[2]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = tid + 256 * i;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (AK) {                       // 8 vectors along k per row, 64 rows
      const int m = m0 + (idx >> 3), k = k0 + (idx & 7) * 4;
      if (m < p.M && k < kend) v = ldg4(p.a + (size_t)m * p.a_rs + k);
    } else {                        // 16 vectors along m per k, 32 k
      const int k = k0 + (idx >> 4), m = m0 + (idx & 15) * 4;
      if (m < p.M && k < kend) v = ldg4(p.a + (size_t)k * p.a_cs + m);
    }
    ra[i] = v;
    v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (BN) {                       // 16 vectors along n per k, 32 k
      const int k = k0 + (idx >> 4), n = n0 + (idx & 15) * 4;
      if (n < p.N && k < kend) v = ldg4(p.b + (size_t)k * p.b_rs + n);
    } else {                        // 8 vectors along k per column, 64 columns
      const int n = n0 + (idx >> 3), k = k0 + (idx & 7) * 4;
      if (n < p.N && k < kend) v = ldg4(p.b + (size_t)n * p.b_cs + k);
    }
    rb[i] = v;
  }
}

template <bool AK, bool BN>
__device__ __forceinline__ void gv_store(int tid, const float4 (&ra)[2], const float4 (&rb)[2], float* As, float* Bs) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = tid + 256 * i;
    if (AK) {
      const int m = idx >> 3, k = (idx & 7) * 4;
      As[(k + 0) * G_STRIDE + m] = ra[i].x; As[(k + 1) * G_STRIDE + m] = ra[i].y;
      As[(k + 2) * G_STRIDE + m] = ra[i].z; As[(k + 3) * G_STRIDE + m] = ra[i].w;
    } else {
      *reinterpret_cast<float4*>(&As[(idx >> 4) * G_STRIDE + (idx & 15) * 4]) = ra[i];
    }
    if (BN) {
      *reinterpret_cast<float4*>(&Bs[(idx >> 4) * G_STRIDE + (idx & 15) * 4]) = rb[i];
    } else {
      const int n = idx >> 3, k = (idx & 7) * 4;
      Bs[(k + 0) * G_STRIDE + n] = rb[i].x; Bs[(k + 1) * G_STRIDE + n] = rb[i].y;
      Bs[(k + 2) * G_STRIDE + n] = rb[i].z; Bs[(k + 3) * G_STRIDE + n] = rb[i].w;
    }
  }
}

template <bool AK, bool BN>
__global__ void __launch_bounds__(256, 3) gemm_vec_kernel(const __grid_constant__ GemmParams p) {
  __shared__ __align__(16) float As[GV_BK * G_STRIDE];
  __shared__ __align__(16) float Bs[GV_BK * G_STRIDE];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * G_BM, n0 = blockIdx.x * G_BN;
  const int kbeg = blockIdx.z * p.k_per_split, kend = min(p.K, kbeg + p.k_per_split);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float4 ra[2], rb[2];
  if (kbeg < kend) gv_load<AK, BN>(p, m0, n0, kbeg, kend, tid, ra, rb);
  for (int k0 = kbeg; k0 < kend; k0 += GV_BK) {
    gv_store<AK, BN>(tid, ra, rb, As, Bs);
    __syncthreads();
    if (k0 + GV_BK < kend) gv_load<AK, BN>(p, m0, n0, k0 + GV_BK, kend, tid, ra, rb);
#pragma unroll
    for (int kk = 0; kk < GV_BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk * G_STRIDE + ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk * G_STRIDE + tx * 4]);
      acc[0][0] = fmaf(a.x, b.x, acc[0][0]); acc[0][1] = fmaf(a.x, b.y, acc[0][1]);
      acc[0][2] = fmaf(a.x, b.z, acc[0][2]); acc[0][3] = fmaf(a.x, b.w, acc[0][3]);
      acc[1][0] = fmaf(a.y, b.x, acc[1][0]); acc[1][1] = fmaf(a.y, b.y, acc[1][1]);
      acc[1][2] = fmaf(a.y, b.z, acc[1][2]); acc[1][3] = fmaf(a.y, b.w, acc[1][3]);
      acc[2][0] = fmaf(a.z, b.x, acc[2][0]); acc[2][1] = fmaf(a.z, b.y, acc[2][1]);
      acc[2][2] = fmaf(a.z, b.z, acc[2][2]); acc[2][3] = fmaf(a.z, b.w, acc[2][3]);
      acc[3][0] = fmaf(a.w, b.x, acc[3][0]); acc[3][1] = fmaf(a.w, b.y, acc[3][1]);
      acc[3][2] = fmaf(a.w, b.z, acc[3][2]); acc[3][3] = fmaf(a.w, b.w, acc[3][3]);
    }
    __syncthreads();
  }
  const bool partial = p.nsplit > 1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.N) continue;
      if (partial) {
        p.ws[((size_t)blockIdx.z * p.M + m) * p.N + n] = acc[i][j];
      } else {
        float v = p.alpha * acc[i][j];
        if (p.bias) v += __ldg(p.bias + n);
        v = apply_act(v, p.act, p.leaky);
        float* o = p.c + (size_t)m * p.c_rs + n;
        if (p.beta != 0.f) v += p.beta * (*o);
        *o = v;
      }
    }
  }
}

// Many small products in one launch (cape_gemm_batch): blockIdx.y = item, the blocks of a row walk its 64 x 64 tiles.
// An item with beta == 1 ACCUMULATES atomically (several items may add into the same C), beta == 0 overwrites.
__global__ void __launch_bounds__(256, 2) gemm_batch_kernel(const GemmParams* __restrict__ items) {
  __shared__ __align__(16) float As[G_BK * G_STRIDE];
  __shared__ __align__(16) float Bs[G_BK * G_STRIDE];
  const GemmParams p = items[blockIdx.y];
  const int mt = (p.M + G_BM - 1) / G_BM, nt = (p.N + G_BN - 1) / G_BN;
  for (int tile = blockIdx.x; tile < mt * nt; tile += gridDim.x)
    gemm_tile(p, (tile / nt) * G_BM, (tile % nt) * G_BN, 0, p.K, 0, p.beta != 0.f ? 2 : 0, As, Bs);
}

// Sum of the split-K partials + epilogue.  The outputs that need a split are few (64 x 64 for the encoder's FC layers)
// and the partials many (a few hundred), so the parallelism has to come from the split axis: 32 consecutive outputs x
// 32 split lanes per CTA, every lane adds its partials in index order, the lanes are added in index order through
// shared memory -- a fixed summation order (deterministic, bit-identical on every replica).
constexpr int GR_EL = 32, GR_ZL = 32;
__global__ void __launch_bounds__(GR_EL * GR_ZL) gemm_reduce_kernel(const __grid_constant__ GemmParams p) {
  __shared__ float red[GR_ZL][GR_EL + 1];
  const long long total = (long long)p.M * p.N;
  const int el = threadIdx.x % GR_EL, zl = threadIdx.x / GR_EL;
  for (long long e0 = (long long)blockIdx.x * GR_EL; e0 < total; e0 += (long long)gridDim.x * GR_EL) {
    const long long e = e0 + el;
    float s = 0.f;
    if (e < total) {
#pragma unroll 4
      for (int z = zl; z < p.nsplit; z += GR_ZL) s += p.ws[(size_t)z * total + e];
    }
    red[zl][el] = s;
    __syncthreads();
    if (zl == 0 && e < total) {
      s = 0.f;
#pragma unroll
      for (int k = 0; k < GR_ZL; ++k) s += red[k][el];
      const int m = (int)(e / p.N), n = (int)(e % p.N);
      float v = p.alpha * s;
      if (p.bias) v += __ldg(p.bias + n);
      v = apply_act(v, p.act, p.leaky);
      float* o = p.c + (size_t)m * p.c_rs + n;
      if (p.beta != 0.f) v += p.beta * (*o);
      *o = v;
    }
    __syncthreads();
  }
}

}  // namespace cape

using namespace cape;

extern "C" int cape_gemm(cape_topology* t, int M, int N, int K, const float* a, int64_t a_rs, int64_t a_cs,
                         const float* b, int64_t b_rs, int64_t b_cs, float* c, int64_t c_rs, const float* bias,
                         int act, float leaky_alpha, float alpha, float beta, void* stream) {
  CAPE_REQUIRE(t && a && b && c, "null pointer");
  CAPE_REQUIRE(M > 0 && N > 0 && K > 0, "empty problem");
  CAPE_REQUIRE(a_cs == 1 || a_rs == 1, "A needs a unit stride");
  CAPE_REQUIRE(b_cs == 1 || b_rs == 1, "B needs a unit stride");
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.a = a; p.a_rs = a_rs; p.a_cs = a_cs;
  p.b = b; p.b_rs = b_rs; p.b_cs = b_cs;
  p.c = c; p.c_rs = c_rs; p.bias = bias; p.act = act; p.leaky = leaky_alpha; p.alpha = alpha; p.beta = beta;
  const int mt = (M + G_BM - 1) / G_BM, nt = (N + G_BN - 1) / G_BN;
  const long long tiles = (long long)mt * nt;
  // the vectorised kernel: worth it from ~1 MB of operands; every 16-byte vector aligned and inside its axis
  // (experiment knob 16 = 1 switches it off)
  const bool a_k = a_cs == 1, b_n = b_cs == 1;
  const bool vec = g_tuning[16] != 1 && (long long)K * (M + N) >= (1LL << 18) && aligned16(a) && aligned16(b) &&
                   (a_k ? (K % 4 == 0 && a_rs % 4 == 0) : (M % 4 == 0 && a_cs % 4 == 0)) &&
                   (b_n ? (N % 4 == 0 && b_rs % 4 == 0) : (K % 4 == 0 && b_cs % 4 == 0));
  const int resident = vec ? 3 : 2;                      // CTAs per SM (launch bounds)
  const int bk = vec ? GV_BK : G_BK;
  long long nsplit = 1;
  if (tiles < (long long)resident * t->sm_count) {
    // one wave of CTAs: half the partials of the former two waves to write and re-read
    nsplit = ((long long)resident * t->sm_count + tiles - 1) / tiles;
    const long long max_by_k = (K + 127) / 128;
    if (nsplit > max_by_k) nsplit = max_by_k;
    const long long per = (long long)M * N * (long long)sizeof(float);
    if (nsplit > 1 && nsplit * per > t->workspace_bytes) nsplit = t->workspace_bytes / per;
    if (nsplit < 1) nsplit = 1;
  }
  int kps = (int)((K + nsplit - 1) / nsplit);
  kps = (kps + bk - 1) / bk * bk;
  nsplit = (K + kps - 1) / kps;
  p.nsplit = (int)nsplit; p.k_per_split = kps; p.ws = (float*)t->workspace;
  CAPE_REQUIRE(mt <= 65535 && nsplit <= 65535, "grid too large");
  dim3 grid(nt, mt, (unsigned)nsplit);
  cudaStream_t st = (cudaStream_t)stream;
  if (!vec) gemm_kernel<<<grid, 256, 0, st>>>(p);
  else if (a_k && b_n) gemm_vec_kernel<true, true><<<grid, 256, 0, st>>>(p);
  else if (a_k) gemm_vec_kernel<true, false><<<grid, 256, 0, st>>>(p);
  else if (b_n) gemm_vec_kernel<false, true><<<grid, 256, 0, st>>>(p);
  else gemm_vec_kernel<false, false><<<grid, 256, 0, st>>>(p);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  if (nsplit > 1) {
    const long long total = (long long)M * N;
    long long blocks = (total + GR_EL - 1) / GR_EL;
    if (blocks > 8LL * t->sm_count) blocks = 8LL * t->sm_count;
    gemm_reduce_kernel<<<(unsigned)blocks, GR_EL * GR_ZL, 0, st>>>(p);
    CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  }
  return 0;
}

extern "C" int cape_gemm_batch(const cape_gemm_item* items_host, int n, void* table_device, int blocks_per_item,
                               void* stream) {
  // items_host != NULL: (re)build the device table (synchronous copy, done once per distinct step schedule);
  // items_host == NULL: launch from the table as it is
  CAPE_REQUIRE(table_device && n > 0 && n <= 65535, "bad arguments");
  if (items_host != nullptr) {
    std::vector<GemmParams> tab((size_t)n);
    for (int i = 0; i < n; ++i) {
      const cape_gemm_item& s = items_host[i];
      CAPE_REQUIRE(s.a && s.b && s.c && s.M > 0 && s.N > 0 && s.K > 0, "bad item");
      CAPE_REQUIRE((s.a_cs == 1 || s.a_rs == 1) && (s.b_cs == 1 || s.b_rs == 1), "operands need a unit stride");
      CAPE_REQUIRE(s.beta == 0.f || s.beta == 1.f, "beta must be 0 (overwrite) or 1 (atomic accumulate)");
      GemmParams& p = tab[i];
      p = GemmParams{};
      p.M = s.M; p.N = s.N; p.K = s.K;
      p.a = s.a; p.a_rs = s.a_rs; p.a_cs = s.a_cs;
      p.b = s.b; p.b_rs = s.b_rs; p.b_cs = s.b_cs;
      p.c = s.c; p.c_rs = s.c_rs; p.alpha = s.alpha; p.beta = s.beta;
      p.nsplit = 1; p.k_per_split = s.K;
    }
    CAPE_CHECK_CUDA(cudaMemcpy(table_device, tab.data(), (size_t)n * sizeof(GemmParams), cudaMemcpyHostToDevice));
    return (int)sizeof(GemmParams);
  }
  if (blocks_per_item < 1) blocks_per_item = 4;
  dim3 grid((unsigned)blocks_per_item, (unsigned)n);
  gemm_batch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const GemmParams*>(table_device));
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}

extern "C" int cape_gemm_item_bytes(void) { return (int)sizeof(GemmParams); }
