// gw_constraint.cu -- PhysicalConstraintLayer on device (graph_weather/models/layers/constraint_layer.py:12-188) in the form
// GraphWeatherForecaster uses it: upsampling_factor = 1, one patch = the whole H x W grid (forecast.py:162-170, 231-246).
//
// In graph terms (node n sits at grid cell cell(n), forecast.py:178-192; src[n] is the row of `hr` / `lr` that the reference's
// graph_to_grid / grid_to_graph round trips leave at node n):
//     additive        y[n] = hr[src n] + lr[src n] - mean_m(hr[src m])                                constraint_layer.py:104-130
//     multiplicative  y[n] = hr[src n] * ( mean_m(lr[src m]) / (mean_m(hr[src m]) + 1e-8) )          :132-160
//     softmax         y[n] = e * (lr[src n] * (1 / e)),  e = exp(exp_factor * hr[src n])               :162-188 (pool of 1)
// Two HBM passes: deterministic column means (per-partition partial sums in double, fixed-order final reduction), then the
// element-wise correction.  Bound: HBM (reads hr twice + lr, writes y: ~4 x B N C x 4 bytes).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/gw_b200.h"
#include "gw_internal.h"

namespace gw {

constexpr int CP = 256;  // node partitions of the mean

// partial[(b * CP + p) * 2C + c] = sum over nodes of partition p of hr[b, src n, c]   (and lr at + C)
__global__ void __launch_bounds__(128) gw_constraint_sums_kernel(const float* __restrict__ hr, const float* __restrict__ lr, int lr_ld,
                                                                 int lr_c, const int32_t* __restrict__ src, long long n_nodes, int C,
                                                                 double* __restrict__ partial) {
  const int p = blockIdx.x, b = blockIdx.y;
  const long long per = (n_nodes + CP - 1) / CP, n0 = p * per, n1 = min(n_nodes, n0 + per);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double sh = 0.0, sl = 0.0;
    for (long long n = n0; n < n1; ++n) {
      const long long r = (long long)b * n_nodes + __ldg(src + n);
      sh += (double)__ldg(hr + r * C + c);
      if (lr) sl += (double)__ldg(lr + r * lr_ld + (c % lr_c));
    }
    partial[((size_t)b * CP + p) * 2 * C + c] = sh;
    partial[((size_t)b * CP + p) * 2 * C + C + c] = sl;
  }
}
// means[b * 2C + c] = (1 / n_nodes) * sum_p partial   (fixed order)
__global__ void gw_constraint_means_kernel(const double* __restrict__ partial, int C, long long n_nodes, float* __restrict__ means) {
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) {
    double s = 0.0;
    for (int p = 0; p < CP; ++p) s += partial[((size_t)b * CP + p) * 2 * C + c];
    means[(size_t)b * 2 * C + c] = (float)(s / (double)n_nodes);
  }
}
__global__ void __launch_bounds__(256) gw_constraint_apply_kernel(int type, const float* __restrict__ hr, const float* __restrict__ lr, int lr_ld,
                                                                  int lr_c, const int32_t* __restrict__ src, long long n_nodes, int C,
                                                                  const float* __restrict__ means, float exp_factor, float* __restrict__ out,
                                                                  int batch) {
  const long long total = (long long)batch * n_nodes * C;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    const long long bn = e / C, b = bn / n_nodes, n = bn - b * n_nodes;
    const long long r = b * n_nodes + __ldg(src + n);
    const float h = __ldg(hr + r * C + c), l = __ldg(lr + r * lr_ld + (c % lr_c));
    float y;
    if (type == GW_CONSTRAINT_ADDITIVE) {
      y = h + (l - means[b * 2 * C + c]);
    } else if (type == GW_CONSTRAINT_MULTIPLICATIVE) {
      y = h * (means[b * 2 * C + C + c] / (means[b * 2 * C + c] + 1e-8f));
    } else {
      const float ex = expf(exp_factor * h);
      y = ex * (l * (1.0f / ex));
    }
    out[e] = y;
  }
}

}  // namespace gw

extern "C" {

int64_t gw_constraint_workspace_bytes(int64_t batch, int32_t channels) {
  return (int64_t)batch * gw::CP * 2 * channels * (int64_t)sizeof(double) + (int64_t)batch * 2 * channels * (int64_t)sizeof(float);
}

int gw_constraint_apply(int32_t type, const float* hr, const float* lr, int32_t lr_ld, int32_t lr_channels, const int32_t* src,
                        float* out, int64_t batch, int64_t n_nodes, int32_t channels, float exp_factor, void* workspace, void* stream) {
  if (!hr || !lr || !src || !out || !workspace) {
    gw::set_error("gw_constraint_apply: null argument");
    return 1;
  }
  if (type != GW_CONSTRAINT_ADDITIVE && type != GW_CONSTRAINT_MULTIPLICATIVE && type != GW_CONSTRAINT_SOFTMAX) {
    gw::set_error("gw_constraint_apply: unknown constraint type");
    return 1;
  }
  if (batch <= 0 || n_nodes <= 0 || channels <= 0 || lr_channels <= 0 || lr_ld < lr_channels || batch > 65535) {
    gw::set_error("gw_constraint_apply: bad sizes");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  double* partial = static_cast<double*>(workspace);
  float* means = reinterpret_cast<float*>(partial + (size_t)batch * gw::CP * 2 * channels);
  if (type != GW_CONSTRAINT_SOFTMAX) {
    gw::gw_constraint_sums_kernel<<<dim3(gw::CP, (unsigned)batch), 128, 0, st>>>(hr, type == GW_CONSTRAINT_MULTIPLICATIVE ? lr : nullptr, lr_ld,
                                                                               lr_channels, src, n_nodes, channels, partial);
    gw::gw_constraint_means_kernel<<<(unsigned)batch, 256, 0, st>>>(partial, channels, n_nodes, means);
    gw::count_launch(2);
  }
  gw::gw_constraint_apply_kernel<<<gw::GRID_SMS * 8, 256, 0, st>>>(type, hr, lr, lr_ld, lr_channels, src, n_nodes, channels, means, exp_factor, out,
                                                        (int)batch);
  gw::count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    gw::set_error(std::string("gw_constraint_apply: ") + cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

}  // extern "C"
