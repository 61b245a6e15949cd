// Topology handle: device-resident ELL operators (the fixed SMPL mesh hierarchy) + workspace.
// Replaces the per-graph tf.SparseTensor construction of lib/models.py:74-79,141-145.
#include "common.cuh"
#include <atomic>
#include <cstring>

namespace cape {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
static std::atomic<long long> g_launches{0};
void count_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launches() { return g_launches.load(std::memory_order_relaxed); }
}  // namespace cape

using namespace cape;

extern "C" const char* cape_last_error(void) { return g_last_error.c_str(); }
extern "C" int cape_abi_version(void) { return CAPE_ABI_VERSION; }
extern "C" int64_t cape_launch_count(void) { return (int64_t)cape::launches(); }

extern "C" int cape_topology_create(int device, cape_topology** out) {
  CAPE_REQUIRE(out != nullptr, "out is null");
  int count = 0;
  CAPE_CHECK_CUDA(cudaGetDeviceCount(&count));
  CAPE_REQUIRE(device >= 0 && device < count, "device index out of range");
  CAPE_CHECK_CUDA(cudaSetDevice(device));
  cape_topology* t = new cape_topology();
  t->device = device;
  cudaDeviceProp prop;
  CAPE_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  t->sm_count = prop.multiProcessorCount;
  if (cudaMalloc(&t->tile_counter, sizeof(unsigned)) != cudaSuccess ||
      cudaMemset(t->tile_counter, 0, sizeof(unsigned)) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
    set_error("cape_topology_create: tile counter allocation failed");
    cudaFree(t->tile_counter);
    delete t;
    return -2;
  }
  *out = t;
  return 0;
}

extern "C" void cape_topology_destroy(cape_topology* t) {
  if (!t) return;
  cudaSetDevice(t->device);
  for (auto& o : t->ops) {
    cudaFree(o.idx);
    cudaFree(o.w);
    cudaFree(o.rowsum);
  }
  if (t->workspace) cudaFree(t->workspace);
  cudaFree(t->tile_counter);
  delete t;
}

extern "C" int cape_topology_add_operator(cape_topology* t, int rows_out, int rows_in, int width,
                                          const int32_t* idx_host, const float* w_host) {
  CAPE_REQUIRE(t && idx_host && w_host, "null pointer");
  CAPE_REQUIRE(rows_out > 0 && rows_in > 0 && width > 0, "bad operator shape");
  // device tables are padded to a width that is a multiple of 4 so kernels can fetch 4 taps with one 16-byte load
  const int width4 = (width + 3) / 4 * 4;
  const size_t n = (size_t)rows_out * width4;
  std::vector<int32_t> idx_p(n, -1);
  std::vector<float> w_p(n, 0.f);
  std::vector<float> rowsum(rows_out, 0.f);
  for (int r = 0; r < rows_out; ++r) {
    double s = 0.0;
    bool ended = false;
    for (int j = 0; j < width; ++j) {
      const int32_t id = idx_host[(size_t)r * width + j];
      if (id < 0) { ended = true; continue; }
      CAPE_REQUIRE(!ended, "ELL rows must be left-packed (no valid slot after an empty one)");
      CAPE_REQUIRE(id < rows_in, "ELL column index out of range");
      s += (double)w_host[(size_t)r * width + j];
      idx_p[(size_t)r * width4 + j] = id;
      w_p[(size_t)r * width4 + j] = w_host[(size_t)r * width + j];
    }
    rowsum[r] = (float)s;
  }
  EllOp o;
  o.rows_out = rows_out; o.rows_in = rows_in; o.width = width4;
  CAPE_CHECK_CUDA(cudaSetDevice(t->device));
  CAPE_CHECK_CUDA(cudaMalloc(&o.idx, n * sizeof(int32_t)));
  CAPE_CHECK_CUDA(cudaMalloc(&o.w, n * sizeof(float)));
  CAPE_CHECK_CUDA(cudaMalloc(&o.rowsum, rows_out * sizeof(float)));
  CAPE_CHECK_CUDA(cudaMemcpy(o.idx, idx_p.data(), n * sizeof(int32_t), cudaMemcpyHostToDevice));
  CAPE_CHECK_CUDA(cudaMemcpy(o.w, w_p.data(), n * sizeof(float), cudaMemcpyHostToDevice));
  CAPE_CHECK_CUDA(cudaMemcpy(o.rowsum, rowsum.data(), rows_out * sizeof(float), cudaMemcpyHostToDevice));
  t->ops.push_back(o);
  return (int)t->ops.size() - 1;
}

extern "C" int cape_topology_reserve_workspace(cape_topology* t, int64_t bytes) {
  CAPE_REQUIRE(t && bytes >= 0, "bad arguments");
  if (bytes <= t->workspace_bytes) return 0;
  CAPE_CHECK_CUDA(cudaSetDevice(t->device));
  CAPE_CHECK_CUDA(cudaDeviceSynchronize());
  if (t->workspace) CAPE_CHECK_CUDA(cudaFree(t->workspace));
  t->workspace = nullptr;
  t->workspace_bytes = 0;
  CAPE_CHECK_CUDA(cudaMalloc(&t->workspace, (size_t)bytes));
  t->workspace_bytes = bytes;
  return 0;
}
