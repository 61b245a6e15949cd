// SMPL linear blend skinning of clothed meshes: the posing step of the reference's demo_full (demos.py:249-331), which
// sets smplx's v_template to the clothed mesh and calls the body model with zero betas (smplx.lbs).  Per mesh:
//   J = J_regressor . v                (the joints regressed from the CLOTHED mesh, as the reference does)
//   R_j = Rodrigues(pose_j)            (smplx.batch_rodrigues)
//   v_posed = v + (R_1..23 - I) . posedirs
//   G_j = G_parent(j) . [R_j | J_j - J_parent(j)],   A_j = G_j - G_j . [J_j, 0]
//   v' = sum_j w_vj A_j . [v_posed, 1]
// Three launches: a per-mesh kernel (joints, rotations, pose feature, kinematic chain -> A), the pose-blend product
// [N, 207] x [207, V*3] on cape_gemm, and a per-vertex skinning kernel over each vertex's non-zero weights.
#include "common.cuh"

namespace cape {

constexpr int SMPL_J = 24, SMPL_PF = 207;
constexpr int SMPL_THREADS = 256;

struct SmplJointParams {
  const float* verts;        // [N, V, 3]
  const float* pose;         // [N, 72] axis-angle
  const int32_t* jreg_ptr;   // [25] CSR row pointers of J_regressor
  const int32_t* jreg_col;
  const float* jreg_val;
  int parents[SMPL_J];       // parents[0] = -1, parents[j] < j
  int V;
  float* pose_feature;       // [N, 207]
  float* A;                  // [N, 24, 12]: rows of the 3x4 relative transform
};

__device__ __forceinline__ float smpl_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(SMPL_THREADS) smpl_joints_kernel(const __grid_constant__ SmplJointParams p) {
  __shared__ float J[SMPL_J][3];
  __shared__ float R[SMPL_J][9];
  __shared__ float G[SMPL_J][12];
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* v = p.verts + (size_t)n * p.V * 3;

  // joint regression: one warp per joint row, lanes stride over its non-zeros, fixed-order shuffle reduction
  for (int j = warp; j < SMPL_J; j += SMPL_THREADS / 32) {
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int k = p.jreg_ptr[j] + lane; k < p.jreg_ptr[j + 1]; k += 32) {
      const float w = __ldg(p.jreg_val + k);
      const float* x = v + (size_t)__ldg(p.jreg_col + k) * 3;
      s0 = fmaf(w, x[0], s0); s1 = fmaf(w, x[1], s1); s2 = fmaf(w, x[2], s2);
    }
    s0 = smpl_warp_sum(s0); s1 = smpl_warp_sum(s1); s2 = smpl_warp_sum(s2);
    if (lane == 0) { J[j][0] = s0; J[j][1] = s1; J[j][2] = s2; }
  }

  // Rodrigues as smplx.batch_rodrigues: angle = |r + 1e-8|, axis = r / angle, R = I + sin K + (1 - cos) K^2
  if (tid < SMPL_J) {
    const float* r = p.pose + (size_t)n * 72 + tid * 3;
    const float rx = r[0], ry = r[1], rz = r[2];
    const float ex = rx + 1e-8f, ey = ry + 1e-8f, ez = rz + 1e-8f;
    const float angle = sqrtf(ex * ex + ey * ey + ez * ez);
    const float x = rx / angle, y = ry / angle, z = rz / angle;
    float s, c;
    sincosf(angle, &s, &c);
    const float t = 1.f - c;
    float* m = R[tid];
    m[0] = 1.f + t * (-(y * y) - z * z); m[1] = -s * z + t * (x * y);    m[2] = s * y + t * (x * z);
    m[3] = s * z + t * (x * y);          m[4] = 1.f + t * (-(x * x) - z * z); m[5] = -s * x + t * (y * z);
    m[6] = -s * y + t * (x * z);         m[7] = s * x + t * (y * z);    m[8] = 1.f + t * (-(x * x) - y * y);
  }
  __syncthreads();

  // pose feature (R_j - I) for the 23 non-root joints, row-major per joint
  for (int i = tid; i < SMPL_PF; i += SMPL_THREADS) {
    const int j = 1 + i / 9, e = i % 9;
    p.pose_feature[(size_t)n * SMPL_PF + i] = R[j][e] - ((e == 0 || e == 4 || e == 8) ? 1.f : 0.f);
  }

  // kinematic chain (24 small products, serial: parents[j] < j was checked when the model was created)
  if (tid == 0) {
    for (int j = 0; j < SMPL_J; ++j) {
      const int par = p.parents[j];
      const float tx = J[j][0] - (par >= 0 ? J[par][0] : 0.f);
      const float ty = J[j][1] - (par >= 0 ? J[par][1] : 0.f);
      const float tz = J[j][2] - (par >= 0 ? J[par][2] : 0.f);
      float* g = G[j];
      if (par < 0) {
        for (int a = 0; a < 3; ++a) {
          g[a * 4 + 0] = R[j][a * 3 + 0]; g[a * 4 + 1] = R[j][a * 3 + 1]; g[a * 4 + 2] = R[j][a * 3 + 2];
        }
        g[3] = tx; g[7] = ty; g[11] = tz;
      } else {
        const float* q = G[par];
        for (int a = 0; a < 3; ++a) {
          for (int b = 0; b < 3; ++b)
            g[a * 4 + b] = q[a * 4 + 0] * R[j][b] + q[a * 4 + 1] * R[j][3 + b] + q[a * 4 + 2] * R[j][6 + b];
          g[a * 4 + 3] = q[a * 4 + 0] * tx + q[a * 4 + 1] * ty + q[a * 4 + 2] * tz + q[a * 4 + 3];
        }
      }
    }
  }
  __syncthreads();

  // relative transforms A_j = G_j - G_j . [J_j, 0]: only the translation column changes
  for (int i = tid; i < SMPL_J * 12; i += SMPL_THREADS) {
    const int j = i / 12, e = i % 12;
    float val = G[j][e];
    if ((e & 3) == 3) {
      const int a = e >> 2;
      val -= G[j][a * 4 + 0] * J[j][0] + G[j][a * 4 + 1] * J[j][1] + G[j][a * 4 + 2] * J[j][2];
    }
    p.A[(size_t)n * SMPL_J * 12 + i] = val;
  }
}

// v' = sum_k w_k A_{j_k} . [v + offset, 1] over the vertex's non-zero weights (idx = -1 ends a row)
__global__ void __launch_bounds__(SMPL_THREADS) smpl_skin_kernel(const float* __restrict__ verts,
                                                                  const float* __restrict__ offsets,
                                                                  const float* __restrict__ A,
                                                                  const int32_t* __restrict__ skin_idx,
                                                                  const float* __restrict__ skin_w, int width, int V,
                                                                  float* __restrict__ out) {
  __shared__ float As[SMPL_J * 12];
  const int n = blockIdx.y;
  for (int i = threadIdx.x; i < SMPL_J * 12; i += blockDim.x) As[i] = A[(size_t)n * SMPL_J * 12 + i];
  __syncthreads();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const size_t base = ((size_t)n * V + v) * 3;
  const float x = verts[base + 0] + offsets[base + 0];
  const float y = verts[base + 1] + offsets[base + 1];
  const float z = verts[base + 2] + offsets[base + 2];
  float T[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) T[e] = 0.f;
  for (int k = 0; k < width; ++k) {
    const int j = __ldg(skin_idx + (size_t)v * width + k);
    if (j < 0) break;
    const float w = __ldg(skin_w + (size_t)v * width + k);
#pragma unroll
    for (int e = 0; e < 12; ++e) T[e] = fmaf(w, As[j * 12 + e], T[e]);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) out[base + a] = T[a * 4 + 0] * x + T[a * 4 + 1] * y + T[a * 4 + 2] * z + T[a * 4 + 3];
}

inline size_t align256(size_t b) { return (b + 255) / 256 * 256; }

}  // namespace cape

struct cape_smpl {
  int device = 0;
  int V = 0;
  int parents[cape::SMPL_J];
  int32_t* jreg_ptr = nullptr;
  int32_t* jreg_col = nullptr;
  float* jreg_val = nullptr;
  float* posedirs = nullptr;    // [207, V*3]
  int32_t* skin_idx = nullptr;  // [V, width]
  float* skin_w = nullptr;
  int width = 0;
  cape_topology* topo = nullptr;  // for cape_gemm (no operators, no workspace)
};

using namespace cape;

extern "C" void cape_smpl_destroy(cape_smpl* s) {
  if (!s) return;
  cudaSetDevice(s->device);
  cudaFree(s->jreg_ptr);
  cudaFree(s->jreg_col);
  cudaFree(s->jreg_val);
  cudaFree(s->posedirs);
  cudaFree(s->skin_idx);
  cudaFree(s->skin_w);
  cape_topology_destroy(s->topo);
  delete s;
}

template <typename T>
static int upload(T** dst, const T* src, size_t n) {
  CAPE_CHECK_CUDA(cudaMalloc(dst, (n > 0 ? n : 1) * sizeof(T)));
  if (n > 0) CAPE_CHECK_CUDA(cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}

extern "C" int cape_smpl_create(int device, int V, const int32_t* jreg_ptr, const int32_t* jreg_col,
                                const float* jreg_val, const float* posedirs, const float* weights,
                                const int32_t* parents, cape_smpl** out) {
  CAPE_REQUIRE(out != nullptr, "out is null");
  *out = nullptr;
  CAPE_REQUIRE(jreg_ptr && jreg_col && jreg_val && posedirs && weights && parents, "null pointer");
  CAPE_REQUIRE(V > 0, "V must be positive");
  CAPE_REQUIRE(jreg_ptr[0] == 0, "J_regressor row pointers must start at 0");
  for (int j = 0; j < SMPL_J; ++j) CAPE_REQUIRE(jreg_ptr[j + 1] >= jreg_ptr[j], "J_regressor row pointers must not decrease");
  const int nnz = jreg_ptr[SMPL_J];
  for (int k = 0; k < nnz; ++k)
    CAPE_REQUIRE(jreg_col[k] >= 0 && jreg_col[k] < V, "J_regressor column index out of range");
  CAPE_REQUIRE(parents[0] == -1, "the root joint's parent must be -1");
  for (int j = 1; j < SMPL_J; ++j)
    CAPE_REQUIRE(parents[j] >= 0 && parents[j] < j, "kinematic tree: parents[j] must lie in [0, j) for j >= 1");
  // skinning weights -> each vertex's non-zero (joint, weight) pairs (exact: only zeros are dropped)
  int width = 1;
  for (int v = 0; v < V; ++v) {
    int c = 0;
    for (int j = 0; j < SMPL_J; ++j) c += weights[(size_t)v * SMPL_J + j] != 0.f;
    width = c > width ? c : width;
  }
  std::vector<int32_t> sidx((size_t)V * width, -1);
  std::vector<float> sw((size_t)V * width, 0.f);
  for (int v = 0; v < V; ++v) {
    int c = 0;
    for (int j = 0; j < SMPL_J; ++j) {
      const float w = weights[(size_t)v * SMPL_J + j];
      if (w != 0.f) { sidx[(size_t)v * width + c] = j; sw[(size_t)v * width + c] = w; ++c; }
    }
  }
  cape_topology* topo = nullptr;
  if (cape_topology_create(device, &topo) != 0) return -2;
  cape_smpl* s = new cape_smpl();
  s->device = device; s->V = V; s->width = width; s->topo = topo;
  for (int j = 0; j < SMPL_J; ++j) s->parents[j] = parents[j];
  int rc = 0;
  if (!rc) rc = upload(&s->jreg_ptr, jreg_ptr, SMPL_J + 1);
  if (!rc) rc = upload(&s->jreg_col, jreg_col, (size_t)nnz);
  if (!rc) rc = upload(&s->jreg_val, jreg_val, (size_t)nnz);
  if (!rc) rc = upload(&s->posedirs, posedirs, (size_t)SMPL_PF * V * 3);
  if (!rc) rc = upload(&s->skin_idx, sidx.data(), sidx.size());
  if (!rc) rc = upload(&s->skin_w, sw.data(), sw.size());
  if (rc) { cape_smpl_destroy(s); return rc; }
  *out = s;
  return 0;
}

extern "C" int64_t cape_smpl_workspace_bytes(const cape_smpl* s, int N) {
  if (!s || N <= 0) { cape::set_error("invalid argument: null model or N <= 0"); return -1; }
  return (int64_t)(align256((size_t)N * SMPL_PF * 4) + align256((size_t)N * SMPL_J * 12 * 4) +
                   align256((size_t)N * s->V * 3 * 4));
}

extern "C" int cape_smpl_pose(cape_smpl* s, int N, const float* verts, const float* pose, float* out, void* workspace,
                              int64_t workspace_bytes, void* stream) {
  CAPE_REQUIRE(s && verts && pose && out && workspace, "null pointer");
  CAPE_REQUIRE(N > 0 && N <= 65535, "N must lie in [1, 65535]");
  CAPE_REQUIRE(aligned16(workspace), "workspace must be 16-byte aligned");
  CAPE_REQUIRE(workspace_bytes >= cape_smpl_workspace_bytes(s, N), "workspace too small (cape_smpl_workspace_bytes)");
  char* ws = static_cast<char*>(workspace);
  float* pf = reinterpret_cast<float*>(ws);
  float* A = reinterpret_cast<float*>(ws + align256((size_t)N * SMPL_PF * 4));
  float* offsets = reinterpret_cast<float*>(ws + align256((size_t)N * SMPL_PF * 4) + align256((size_t)N * SMPL_J * 12 * 4));
  cudaStream_t st = (cudaStream_t)stream;
  SmplJointParams p{};
  p.verts = verts; p.pose = pose;
  p.jreg_ptr = s->jreg_ptr; p.jreg_col = s->jreg_col; p.jreg_val = s->jreg_val;
  for (int j = 0; j < SMPL_J; ++j) p.parents[j] = s->parents[j];
  p.V = s->V; p.pose_feature = pf; p.A = A;
  smpl_joints_kernel<<<N, SMPL_THREADS, 0, st>>>(p);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  const int cols = s->V * 3;
  const int rc = cape_gemm(s->topo, N, cols, SMPL_PF, pf, SMPL_PF, 1, s->posedirs, cols, 1, offsets, cols, nullptr,
                           CAPE_ACT_NONE, 0.f, 1.f, 0.f, stream);
  if (rc != 0) return rc;
  dim3 grid((unsigned)((s->V + SMPL_THREADS - 1) / SMPL_THREADS), (unsigned)N);
  smpl_skin_kernel<<<grid, SMPL_THREADS, 0, st>>>(verts, offsets, A, s->skin_idx, s->skin_w, s->width, s->V, out);
  CAPE_CHECK_CUDA(cudaGetLastError());
  cape::count_launches(1);
  return 0;
}
