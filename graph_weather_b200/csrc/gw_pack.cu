// gw_pack.cu -- packing of nn.Linear weights (once per weight set; every step for the training step's W and W^T images, scale taken
// on the device) into the operand images the tensor-core chain kernel (gw_tc3.cu) streams:
// fp16 hi|lo (fp32-faithful mode) or bf16, K-major, SWIZZLE_128B, one contiguous panel per 64-wide K chunk, power-of-two
// pre-scaled, output rows and K columns permuted inside every group of 32 (perm32) -- the feature order of the chain kernel's
// wgmma accumulator fragments, see gw_tc3.cu.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "gw_internal.h"

namespace gw {

// ------------------------------------------------------------------------------------------------------------------
// weight packing (one-off per weight set)
// ------------------------------------------------------------------------------------------------------------------
static inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
// rows of a packed image: N padded to 64 (the kernel's 64-column epilogue chunks; the forecast's 78-column output layer has 128)
int tc_packed_rows(int N_src) { return round_up(N_src, 64); }
size_t tc_packed_bytes(int K_src, int N_src, int parts) {
  return (size_t)(round_up(K_src, 64) / 64) * parts * tc_packed_rows(N_src) * 128;
}

// dst image: for chunk kc, part p: panel of N rows x 128 B; element (n, k): 16B chunk ((k%64)/8) ^ (n&7), half k%8
// perm32 (wgmma accumulator fragments: a thread owns 8 consecutive features of a row): inside every group of 32,
// packed position a = 8g + 2c + e holds logical index 8c + 2g + e.
__host__ __device__ inline int perm32_f(int a) { return (a & ~31) | (8 * ((a >> 1) & 3) + 2 * ((a >> 3) & 3) + (a & 1)); }
__global__ void gw_pack_weights_kernel(const float* __restrict__ W, int ldw, int K_src, int N_src, int Kp, int Np,
                                       float wscale, int parts, uint8_t* __restrict__ dst, const float* __restrict__ amax_dev) {
  if (amax_dev) wscale = tc_weight_scale(*amax_dev, parts);
  const size_t total = (size_t)Np * Kp;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(e / Kp), k = (int)(e % Kp);
    const int ns = perm32_f(n), ks = perm32_f(k);  // (rows padded to 64, K is always a multiple of 64)
    const float w = (ns < N_src && ks < K_src) ? W[(size_t)ns * ldw + ks] * wscale : 0.f;
    const int kc = k >> 6, kk = k & 63;
    const size_t panel = (size_t)Np * 128;
    const size_t off = (size_t)n * 128 + (size_t)((((kk >> 3) ^ (n & 7)) << 4) + ((kk & 7) << 1));
    if (parts == 2) {
      const __half hi = __float2half_rn(w);
      const __half lo = __float2half_rn(w - __half2float(hi));
      *reinterpret_cast<__half*>(dst + (size_t)(kc * 2 + 0) * panel + off) = hi;
      *reinterpret_cast<__half*>(dst + (size_t)(kc * 2 + 1) * panel + off) = lo;
    } else {
      *reinterpret_cast<__nv_bfloat16*>(dst + (size_t)kc * panel + off) = __float2bfloat16_rn(w);
    }
  }
}

cudaError_t launch_pack_weights(const float* W, int ldw, int K_src, int N_src, float wscale, int parts, void* dst,
                                cudaStream_t stream, const float* amax_dev) {
  const int Kp = round_up(K_src, 64), Np = tc_packed_rows(N_src);
  gw_pack_weights_kernel<<<256, 256, 0, stream>>>(W, ldw, K_src, N_src, Kp, Np, wscale, parts, static_cast<uint8_t*>(dst), amax_dev);
  count_launch();
  return cudaGetLastError();
}

__global__ void gw_absmax_kernel(const float* __restrict__ W, int ldw, int K_src, int N_src, float* out_max) {
  float m = 0.f;
  const size_t total = (size_t)N_src * K_src;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(W[(e / K_src) * (size_t)ldw + (e % K_src)]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out_max), __float_as_int(m));  // m >= 0: int order == float order
}

cudaError_t launch_absmax(const float* W, int ldw, int K_src, int N_src, float* out_max, cudaStream_t stream) {
  gw_absmax_kernel<<<64, 256, 0, stream>>>(W, ldw, K_src, N_src, out_max);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_pack_image(const float* W, int ldw, int K_src, int N_src, int parts, void* img, float* wamax, cudaStream_t stream) {
  cudaError_t e = cudaMemsetAsync(wamax, 0, sizeof(float), stream);
  if (e == cudaSuccess) e = launch_absmax(W, ldw, K_src, N_src, wamax, stream);
  if (e == cudaSuccess) e = launch_pack_weights(W, ldw, K_src, N_src, 1.f, parts, img, stream, wamax);
  return e;
}

TcWeights tc_weights(const void* img, int K_src, int N_src, float wamax, int parts) {
  TcWeights w;
  w.p = img, w.K = round_up(K_src, 64), w.N = round_up(N_src, 16), w.N32 = tc_packed_rows(N_src), w.n_valid = N_src;
  w.winv = 1.f / tc_weight_scale(wamax, parts), w.gain = (float)K_src * wamax;
  return w;
}

}  // namespace gw
