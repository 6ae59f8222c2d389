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
// The backward (gw_constraint_backward, below) is one column-sum pass over dy (and hr) plus one pass over the rows through the
// CSR of src: ~5 x B N C x 4 bytes.
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

// ---- backward ---------------------------------------------------------------------------------------------------------------------
// With cnt(r) = #{n : src n = r} and column sums over all nodes (per sample and channel):
//     additive        d_hr[r] = sum_{src n = r} dy[n] - cnt(r)/N S,                   d_lr[r] = sum_{src n = r} dy[n],   S = sum_n dy[n]
//     multiplicative  d_hr[r] = rho sum_{src n = r} dy[n] - cnt(r)/N ML/(MH+eps)^2 T, d_lr[r] = cnt(r)/N T/(MH+eps),     T = sum_n dy[n] hr[src n]
//     softmax         torch's autograd of constraint_layer.py:172-187 op by op in fp32 per node, then summed per row
// Rows no node reads get 0; a shared row sums its nodes in ascending node order (CSR of src built by a stable sort).  Column sums as
// in the forward: per-partition double partials, fixed-order finish.  No atomics: bit for bit repeatable.

// partial[(b * CP + p) * C + c] = sum over nodes of partition p of dy[b, n, c] (* hr[b, src n, c] if hr)
__global__ void __launch_bounds__(128) gw_constraint_grad_sums_kernel(const float* __restrict__ dy, const float* __restrict__ hr,
                                                                      const int32_t* __restrict__ src, long long n_nodes, int C,
                                                                      double* __restrict__ partial) {
  const int p = blockIdx.x, b = blockIdx.y;
  const long long per = (n_nodes + CP - 1) / CP, n0 = p * per, n1 = min(n_nodes, n0 + per);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double s = 0.0;
    for (long long n = n0; n < n1; ++n) {
      const double g = (double)__ldg(dy + ((long long)b * n_nodes + n) * C + c);
      s += hr ? g * (double)__ldg(hr + ((long long)b * n_nodes + __ldg(src + n)) * C + c) : g;
    }
    partial[((size_t)b * CP + p) * C + c] = s;
  }
}
// coef[b * 2C + c] = per-node coefficient of d_hr, coef[b * 2C + C + c] = that of d_lr (both times cnt(r)); rho[b * C + c]
__global__ void gw_constraint_grad_coef_kernel(int type, const double* __restrict__ partial, int C, long long n_nodes,
                                               const float* __restrict__ means, double* __restrict__ coef, float* __restrict__ rho) {
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    double s = 0.0;
    for (int p = 0; p < CP; ++p) s += partial[((size_t)b * CP + p) * C + c];
    double kh = -s / (double)n_nodes, kl = 0.0;
    if (type == GW_CONSTRAINT_MULTIPLICATIVE) {
      const float mh = means[(size_t)b * 2 * C + c], ml = means[(size_t)b * 2 * C + C + c];
      const float den = mh + 1e-8f;  // the forward's denominator and ratio, bit for bit
      rho[(size_t)b * C + c] = ml / den;
      kh = -(double)ml / ((double)den * (double)den) * s / (double)n_nodes;
      kl = s / (double)den / (double)n_nodes;
    }
    coef[(size_t)b * 2 * C + c] = kh;
    coef[(size_t)b * 2 * C + C + c] = kl;
  }
}
__global__ void __launch_bounds__(256) gw_constraint_bwd_rows_kernel(int type, const float* __restrict__ dy, const float* __restrict__ hr,
                                                                     const float* __restrict__ lr, int lr_ld, const int32_t* __restrict__ perm,
                                                                     const int32_t* __restrict__ ptr, long long n_nodes, int C,
                                                                     const double* __restrict__ coef, const float* __restrict__ rho,
                                                                     float exp_factor, float* __restrict__ d_hr, float* __restrict__ d_lr,
                                                                     int batch) {
  const long long total = (long long)batch * n_nodes * C;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C);
    const long long br = e / C, b = br / n_nodes, r = br - b * n_nodes;
    const int j0 = __ldg(ptr + r), j1 = __ldg(ptr + r + 1);
    float gh = 0.f, gl = 0.f;
    if (j1 > j0) {
      const float* dyb = dy + b * n_nodes * C + c;
      double sh = 0.0, sl = 0.0;
      if (type == GW_CONSTRAINT_SOFTMAX) {
        const float h = __ldg(hr + e), l = __ldg(lr + br * lr_ld + c);
        const float ex = expf(__fmul_rn(exp_factor, h)), rc = 1.0f / ex, q = __fmul_rn(l, rc), rr = __fmul_rn(rc, rc);
        for (int j = j0; j < j1; ++j) {
          const float g = __ldg(dyb + (long long)__ldg(perm + j) * C);
          const float d_ratio = __fmul_rn(g, ex);
          const float d_e = __fadd_rn(__fmul_rn(g, q), -__fmul_rn(__fmul_rn(d_ratio, l), rr));
          sh += (double)__fmul_rn(__fmul_rn(d_e, ex), exp_factor);
          sl += (double)__fmul_rn(d_ratio, rc);
        }
      } else {
        for (int j = j0; j < j1; ++j) sh += (double)__ldg(dyb + (long long)__ldg(perm + j) * C);
        const double cnt = (double)(j1 - j0), kh = coef[b * 2 * C + c], kl = coef[b * 2 * C + C + c];
        if (type == GW_CONSTRAINT_ADDITIVE) {
          sl = sh;
          sh += cnt * kh;
        } else {
          sl = cnt * kl;
          sh = (double)rho[b * C + c] * sh + cnt * kh;
        }
      }
      gh = (float)sh, gl = (float)sl;
    }
    d_hr[e] = gh;
    if (d_lr) d_lr[e] = gl;
  }
}

static size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// workspace: [forward sums + means][grad partials][coef][rho][perm][ptr][sort]
struct BwdWs {
  size_t fwd, partial, coef, rho, perm, ptr, sort, total;
};
static BwdWs bwd_ws_layout(int64_t batch, int64_t n_nodes, int32_t channels) {
  BwdWs w;
  w.fwd = 0;
  w.partial = w.fwd + align256((size_t)gw_constraint_workspace_bytes(batch, channels));
  w.coef = w.partial + align256((size_t)batch * CP * channels * sizeof(double));
  w.rho = w.coef + align256((size_t)batch * 2 * channels * sizeof(double));
  w.perm = w.rho + align256((size_t)batch * channels * sizeof(float));
  w.ptr = w.perm + align256((size_t)n_nodes * sizeof(int32_t));
  w.sort = w.ptr + align256((size_t)(n_nodes + 1) * sizeof(int32_t));
  w.total = w.sort + align256(sort_csr_workspace_bytes((int)n_nodes));
  return w;
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

int64_t gw_constraint_backward_workspace_bytes(int64_t batch, int64_t n_nodes, int32_t channels) {
  if (batch <= 0 || n_nodes <= 0 || n_nodes >= INT32_MAX || channels <= 0) return 0;
  return (int64_t)gw::bwd_ws_layout(batch, n_nodes, channels).total;
}

int gw_constraint_backward(int32_t type, const float* dy, const float* hr, const float* lr, int32_t lr_ld, int32_t lr_channels, const int32_t* src,
                           float* d_hr, float* d_lr, int64_t batch, int64_t n_nodes, int32_t channels, float exp_factor, void* workspace,
                           void* stream) {
  if (!dy || !hr || !lr || !src || !d_hr || !workspace) {
    gw::set_error("gw_constraint_backward: null argument");
    return 1;
  }
  if (type != GW_CONSTRAINT_ADDITIVE && type != GW_CONSTRAINT_MULTIPLICATIVE && type != GW_CONSTRAINT_SOFTMAX) {
    gw::set_error("gw_constraint_backward: unknown constraint type");
    return 1;
  }
  if (batch <= 0 || n_nodes <= 0 || n_nodes >= INT32_MAX || channels <= 0 || lr_ld < lr_channels || batch > 65535) {
    gw::set_error("gw_constraint_backward: bad sizes");
    return 1;
  }
  if (lr_channels != channels) {
    gw::set_error("gw_constraint_backward: lr_channels must equal channels (the backward of the channel repeat is not built)");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const gw::BwdWs L = gw::bwd_ws_layout(batch, n_nodes, channels);
  uint8_t* w = static_cast<uint8_t*>(workspace);
  double* fwd_partial = reinterpret_cast<double*>(w + L.fwd);
  float* means = reinterpret_cast<float*>(fwd_partial + (size_t)batch * gw::CP * 2 * channels);
  double* partial = reinterpret_cast<double*>(w + L.partial);
  double* coef = reinterpret_cast<double*>(w + L.coef);
  float* rho = reinterpret_cast<float*>(w + L.rho);
  int32_t* perm = reinterpret_cast<int32_t*>(w + L.perm);
  int32_t* ptr = reinterpret_cast<int32_t*>(w + L.ptr);
  // rows -> the nodes that read them, ascending (stable sort)
  cudaError_t e = gw::launch_sort_csr(src, (int)n_nodes, (int)n_nodes, perm, ptr, w + L.sort, L.total - L.sort, st);
  if (e == cudaSuccess && type != GW_CONSTRAINT_SOFTMAX) {
    if (type == GW_CONSTRAINT_MULTIPLICATIVE) {  // the forward's means, recomputed by its own kernels
      gw::gw_constraint_sums_kernel<<<dim3(gw::CP, (unsigned)batch), 128, 0, st>>>(hr, lr, lr_ld, lr_channels, src, n_nodes, channels, fwd_partial);
      gw::gw_constraint_means_kernel<<<(unsigned)batch, 256, 0, st>>>(fwd_partial, channels, n_nodes, means);
      gw::count_launch(2);
    }
    gw::gw_constraint_grad_sums_kernel<<<dim3(gw::CP, (unsigned)batch), 128, 0, st>>>(dy, type == GW_CONSTRAINT_MULTIPLICATIVE ? hr : nullptr, src,
                                                                                    n_nodes, channels, partial);
    gw::gw_constraint_grad_coef_kernel<<<(unsigned)batch, 128, 0, st>>>(type, partial, channels, n_nodes, means, coef, rho);
    gw::count_launch(2);
  }
  if (e == cudaSuccess) {
    gw::gw_constraint_bwd_rows_kernel<<<gw::GRID_SMS * 8, 256, 0, st>>>(type, dy, hr, lr, lr_ld, perm, ptr, n_nodes, channels, coef, rho, exp_factor,
                                                                       d_hr, d_lr, (int)batch);
    gw::count_launch();
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) {
    gw::set_error(std::string("gw_constraint_backward: ") + cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

}  // extern "C"
