// gw_loss.cu -- the loss boundary of the forward (SURVEY 8(f) row 2, forward half): NormalizedMSELoss.forward
// (graph_weather/models/losses.py:46-94) as one HBM-bound reduction.
//
//   loss = mean_{b,n} [ w(n) * mean_f ( (pred - target)^2 [/ feature_variance_f] ) ]        w(n) = cos(lat of grid row n / num_lon)
//
// The kernel returns the SUM over the local rows (sum_{b,n} w(n) * mean_f(...)), in double, so that data-parallel ranks
// exchange one scalar (all-reduce of the sums, divide by the global B*N) instead of all-gathering 162 MB of outputs per rank.
// Bound: HBM -- 2 * 4 * B * N * F bytes read once (324 MB at 1 deg / batch 8), no reuse.  Deterministic: one warp per row,
// fixed-shape tree inside the CTA, per-CTA partials summed in index order by a second, single-CTA launch.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gw_b200.h"
#include "gw_internal.h"

namespace gw {

constexpr int LOSS_THREADS = 256, LOSS_WARPS = LOSS_THREADS / 32;

__global__ void __launch_bounds__(LOSS_THREADS) gw_loss_partial_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                                                      const float* __restrict__ inv_var, const float* __restrict__ node_w,
                                                                      long long rows, int n_nodes, int F, double* __restrict__ partial) {
  __shared__ double wsum[LOSS_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float inv_f = 1.0f / (float)F;
  double acc = 0.0;
  const long long stride = (long long)gridDim.x * LOSS_WARPS;
  for (long long r0 = (long long)blockIdx.x * LOSS_WARPS + warp; r0 < rows; r0 += 4 * stride) {
    float s[4] = {0.f, 0.f, 0.f, 0.f};  // four rows per warp in flight (independent loads), each reduced on its own
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const long long r = r0 + u * stride;
      if (r < rows) {
        const float* p = pred + r * F;
        const float* t = target + r * F;
        for (int f = lane; f < F; f += 32) {  // consecutive lanes read consecutive floats of the row
          const float d = __ldg(p + f) - __ldg(t + f);
          const float q = d * d;
          s[u] += inv_var ? q * __ldg(inv_var + f) : q;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
      const long long r = r0 + u * stride;
      if (r < rows) acc += (double)(s[u] * inv_f * __ldg(node_w + (int)(r % n_nodes)));  // same value in every lane
    }
  }
  if (lane == 0) wsum[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int w = 0; w < LOSS_WARPS; ++w) tot += wsum[w];
    partial[blockIdx.x] = tot;
  }
}

__global__ void gw_loss_final_kernel(const double* __restrict__ partial, int n, double* __restrict__ out) {
  // one warp; lane i adds partial[i], partial[i + 32], ... in index order, then a fixed shuffle tree: the same result on every run
  double tot = 0.0;
  for (int i = threadIdx.x; i < n; i += 32) tot += partial[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
  if (threadIdx.x == 0) *out = tot;
}

constexpr int LOSS_GRID = GRID_SMS * 8;

// d(sum) / d pred[b, n, f] * scale = scale * w(n) * 2 (pred - target) * inv_var(f) / F          (losses.py:70-94 differentiated)
__global__ void __launch_bounds__(256) gw_loss_grad_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                                           const float* __restrict__ inv_variance, const float* __restrict__ node_weight,
                                                           long long rows, int n_nodes, int F, const float* __restrict__ scale_dev, float scale,
                                                           float* __restrict__ grad) {
  const float sc = (scale_dev ? __ldg(scale_dev) : 1.f) * scale * 2.f / (float)F;
  const long long total = rows * F;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / F;
    const int f = (int)(e - r * F);
    const float w = __ldg(node_weight + (int)(r % n_nodes));
    const float iv = inv_variance ? __ldg(inv_variance + f) : 1.f;
    grad[e] = sc * w * iv * (__ldg(pred + e) - __ldg(target + e));
  }
}

}  // namespace gw

extern "C" {

int gw_normalized_mse_loss_grad(const float* pred, const float* target, const float* inv_variance, const float* node_weight, int64_t batch,
                                int64_t n_nodes, int32_t n_features, const float* scale_dev, float scale, float* grad_pred, void* stream) {
  if (!pred || !target || !node_weight || !grad_pred) {
    gw::set_error("gw_normalized_mse_loss_grad: null argument");
    return 1;
  }
  if (batch <= 0 || n_nodes <= 0 || n_features <= 0 || n_nodes > 0x7fffffffLL) {
    gw::set_error("gw_normalized_mse_loss_grad: bad shape");
    return 1;
  }
  gw::gw_loss_grad_kernel<<<gw::GRID_SMS * 8, 256, 0, (cudaStream_t)stream>>>(pred, target, inv_variance, node_weight, (long long)batch * n_nodes, (int)n_nodes,
                                                                   n_features, scale_dev, scale, grad_pred);
  gw::count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    gw::set_error(std::string("loss gradient kernel failed to launch: ") + cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

int64_t gw_loss_workspace_bytes(void) { return (int64_t)gw::LOSS_GRID * (int64_t)sizeof(double); }

int gw_normalized_mse_loss_sum(const float* pred, const float* target, const float* inv_variance, const float* node_weight, int64_t batch,
                               int64_t n_nodes, int32_t n_features, double* sum_out, void* workspace, void* stream) {
  if (!pred || !target || !node_weight || !sum_out || !workspace) {
    gw::set_error("gw_normalized_mse_loss_sum: null argument");
    return 1;
  }
  if (batch <= 0 || n_nodes <= 0 || n_features <= 0 || n_nodes > 0x7fffffffLL) {
    gw::set_error("gw_normalized_mse_loss_sum: bad shape");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = (long long)batch * n_nodes;
  long long want = (rows + gw::LOSS_WARPS - 1) / gw::LOSS_WARPS;
  const int grid = (int)(want < gw::LOSS_GRID ? want : gw::LOSS_GRID);
  gw::gw_loss_partial_kernel<<<grid, gw::LOSS_THREADS, 0, st>>>(pred, target, inv_variance, node_weight, rows, (int)n_nodes, n_features,
                                                              static_cast<double*>(workspace));
  gw::gw_loss_final_kernel<<<1, 32, 0, st>>>(static_cast<const double*>(workspace), grid, sum_out);
  gw::count_launch(2);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    gw::set_error(std::string("loss kernels failed to launch: ") + cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

}  // extern "C"
