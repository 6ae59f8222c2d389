// gw_wgrad_tc.cu -- weight gradient of a Linear layer on Hopper tensor cores (wgmma), for the training step of the tensor-core
// precisions (gw_train.cu):
//     dW[o, k] += sum_r dY[r, o] . A(r, k)        db[o] += sum_r dY[r, o]
// over R = batch x rows_per_sample rows (up to ~3.6 M: the decoder's edges at 1 degree, batch 8).  The reduction runs over the
// rows, so each CTA takes a contiguous range of them and forms a partial dW block; a second kernel sums the partials in a fixed
// order.  No float atomics: the weight gradients are repeatable bit for bit.
//
// Layout of the work (one CTA = 2 consumer warpgroups = 256 threads, 1 CTA per SM):
//   * output block: 128 rows o (warpgroup w owns 64 w .. 64 w + 63, a 64 x NW fp32 accumulator in registers, NW = K rounded up
//     to 64 <= 256) x all K columns; gridDim.y = ceil(N / 128) blocks of o, gridDim.x = row ranges.  A wider K (the encoder's
//     621 input features) runs as blocks of 256 columns, each a launch of its own over all rows, one after the other.
//   * per 64-row chunk r0 .. r0 + 63 the threads read dY[r, o] and A(r, k) (coalesced along o / k), split them to fp16 hi/lo (or
//     round to bf16) and store them TRANSPOSED into two K-major SWIZZLE_128B images [o][r] and [k][r] -- the layout of the chain
//     kernel's operands (gw_tc3.cu), so the same GMMA descriptors apply: D[o, k] += Y^T[o, r] . (A^T[k, r])^T.  A thread loads 8
//     rows x 4 columns and writes, per column, one 16-byte swizzle chunk (8 rows): the 8 lanes of a store phase hit 8 different
//     chunks of one 128-byte row, no bank conflicts.
//   * the images are double buffered: chunk c + 1 is loaded and converted while the wgmma of chunk c run.
//   * fp32-faithful mode: both operands are scaled by powers of two from their absmax (one pass each, before the kernel) into
//     [2^14, 2^15), so the lo parts of ~1e-8 gradients stay normal; the accumulator is unscaled exactly in the epilogue.
//   * the bias gradient is the fp32 column sum of the dY values the CTA loads anyway (8-lane shuffle, fixed order).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "gw_internal.h"
#include "gw_ops.h"
#include "gw_tc_ptx.cuh"

namespace gw {
namespace wgt {

constexpr int RC = 64;                      // rows per chunk (the K of four m64nNk16 steps)
constexpr int OB = 128;                     // o rows per CTA
constexpr int THREADS = 256;
constexpr int Y_HALF = OB * 128;            // [128 o][64 r] 16-bit
constexpr int A_HALF = 256 * 128;           // [256 k][64 r] 16-bit
constexpr int STAGE = 2 * (Y_HALF + A_HALF);  // hi | lo of both images
constexpr int SMEM_BYTES = 2 * STAGE + 1024;  // two stages + alignment slack
static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB per-CTA shared memory limit");

struct Args {
  const float* dY;
  int ldy, N, K;
  RowSrc a;
  int rows, batch;
  long long R;
  int rows_per_cta;  // multiple of RC
  float* part;       // [gridDim.x][N][K]
  float* part_b;     // [gridDim.x][N]
  const float* amax; // [2]: max|dY|, max|A| (fp32-faithful mode)
  int32_t* status;
};

__device__ __forceinline__ float pow2_fit(float m) {  // power of two s with s m in [2^14, 2^15); 1 for zero / non-finite m
  if (!(m > 0.f) || !(m < 3.0e38f)) return 1.f;
  int e = (int)((__float_as_uint(m) >> 23) & 0xffu) - 127;
  e = e < -110 ? -110 : e;
  return __uint_as_float((uint32_t)(127 + 14 - e) << 23);
}

// 8 rows x 4 columns of a row-major tensor -> v[row][col]; zero beyond `nrows` rows / `width` columns.  vec: rows are 16-byte aligned
template <class RowPtr>
__device__ __forceinline__ void load_8x4(RowPtr rowp, int nrows, int c, int width, bool vec, float (&v)[8][4]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (j < nrows) {
      const float* p = rowp(j) + c;
      if (vec && c + 4 <= width) {
        const float4 f = __ldg(reinterpret_cast<const float4*>(p));
        v[j][0] = f.x, v[j][1] = f.y, v[j][2] = f.z, v[j][3] = f.w;
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) v[j][i] = (c + i < width) ? __ldg(p + i) : 0.f;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) v[j][i] = 0.f;
    }
  }
}

// v[8 rows][4 columns] (times s) -> images: column c + i is image row n, the 8 rows are 16-bit elements 8 g .. 8 g + 7 of it
template <bool SPLIT>
__device__ __forceinline__ void store_t(uint32_t img, uint32_t lo_off, int c, int g, const float (&v)[8][4], float s) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int n = c + i;
    const uint32_t addr = img + (uint32_t)n * 128u + (uint32_t)(((g ^ (n & 7)) & 7) << 4);
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a0 = v[2 * j][i] * s, a1 = v[2 * j + 1][i] * s;
      if (SPLIT) {
        const __half2 hh = __floats2half2_rn(a0, a1);
        const float2 hf = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
        hi[j] = *reinterpret_cast<const uint32_t*>(&hh), lo[j] = *reinterpret_cast<const uint32_t*>(&ll);
      } else {
        const __nv_bfloat162 bb = __floats2bfloat162_rn(a0, a1);
        hi[j] = *reinterpret_cast<const uint32_t*>(&bb);
      }
    }
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(hi[0]), "r"(hi[1]), "r"(hi[2]), "r"(hi[3]) : "memory");
    if (SPLIT)
      asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr + lo_off), "r"(lo[0]), "r"(lo[1]), "r"(lo[2]), "r"(lo[3]) : "memory");
  }
}

template <bool SPLIT, int NW>
__global__ void __launch_bounds__(THREADS, 1) gw_wgrad_tc_kernel(const __grid_constant__ Args a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane & 7, q = lane >> 3;  // staging: row group g (8 rows) x column quad q of the warp's 16 columns
  const int o0 = blockIdx.y * OB;
  const long long rb = (long long)blockIdx.x * a.rows_per_cta;
  const long long re = rb + a.rows_per_cta < a.R ? rb + a.rows_per_cta : a.R;
  const int nchunks = rb < re ? (int)((re - rb + RC - 1) / RC) : 0;
  float sy = 1.f, sa = 1.f;
  if (SPLIT) {
    const float my = __ldg(a.amax), ma = __ldg(a.amax + 1);
    if (!(my < 3.0e38f) || !(ma < 3.0e38f)) {
      if (a.status && threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0) atomicOr(a.status, 8);  // non-finite gradient / activation
    }
    sy = pow2_fit(my), sa = pow2_fit(ma);
  }
  const bool vec_y = ((a.ldy & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.dY) & 15) == 0);
  const bool vec_a = ((a.a.ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.a.base + a.a.col0) & 15) == 0);
  const bool bcast = a.a.kind == SRC_BCAST;
  const int cy = 4 * (4 * warp + q);  // my dY column quad (o0 + cy .. + 3): 8 warps x 4 quads = 128 columns
  float bsum[4] = {0.f, 0.f, 0.f, 0.f};

  auto stage = [&](int c, int buf) {
    const uint32_t st = sbase + (uint32_t)buf * STAGE;
    const long long r0 = rb + (long long)c * RC + 8 * g;
    const int nr = re - r0 >= 8 ? 8 : (re - r0 > 0 ? (int)(re - r0) : 0);
    float v[8][4];
    load_8x4([&](int j) { return a.dY + (size_t)(r0 + j) * (size_t)a.ldy + o0; }, nr, cy, a.N - o0, vec_y && ((o0 & 3) == 0), v);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) bsum[i] += v[j][i];
    store_t<SPLIT>(st, Y_HALF, cy, g, v, sy);
    for (int ck = 4 * (4 * warp + q); ck < NW; ck += 128) {  // A columns: 32 quads per pass over the 8 warps
      load_8x4(
          [&](int j) {
            const long long r = r0 + j;
            const long long b = r / a.rows, i = r - b * a.rows;
            return a.a.base + (size_t)(bcast ? i : b * (long long)a.a.src_rows + i) * (size_t)a.a.ld + a.a.col0;
          },
          nr, ck, a.K, vec_a, v);
      store_t<SPLIT>(st + 2 * Y_HALF, A_HALF, ck, g, v, sa);
    }
    fence_proxy_async();  // generic-proxy stores -> visible to the wgmma (async proxy)
  };

  float d[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) d[i] = 0.f;
  const int wg = warp >> 2;
  if (nchunks > 0) stage(0, 0);
  __syncthreads();
  for (int c = 0; c < nchunks; ++c) {
    const uint32_t st = sbase + (uint32_t)(c & 1) * STAGE;
    const uint32_t y_hi = st + (uint32_t)wg * 64u * 128u, y_lo = y_hi + Y_HALF;
    const uint32_t a_hi = st + 2 * Y_HALF, a_lo = a_hi + A_HALF;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      Wgmma<NW, !SPLIT>::mma(d, gmma_desc(y_hi + 32 * ks), gmma_desc(a_hi + 32 * ks), 1);
      if (SPLIT) {
        Wgmma<NW, !SPLIT>::mma(d, gmma_desc(y_lo + 32 * ks), gmma_desc(a_hi + 32 * ks), 1);
        Wgmma<NW, !SPLIT>::mma(d, gmma_desc(y_hi + 32 * ks), gmma_desc(a_lo + 32 * ks), 1);
      }
    }
    wgmma_commit();
    if (c + 1 < nchunks) stage(c + 1, (c + 1) & 1);  // overlaps the wgmma of chunk c
    wgmma_wait<0>();
    fence_operand(d);
    __syncthreads();  // both warpgroups are done with stage c & 1 before it is refilled
  }
  // partial block -> workspace: thread t of warp q4 holds (o = 16 q4 + t/4 + 8 m, k = 8 j + 2 (t % 4) + e) of its warpgroup's 64 rows
  const float inv = (1.f / sy) * (1.f / sa);
  const int q4 = warp & 3;
  float* part = a.part + (size_t)blockIdx.x * a.N * a.K;
#pragma unroll
  for (int m = 0; m < 2; ++m) {
    const int o = o0 + 64 * wg + 16 * q4 + (lane >> 2) + 8 * m;
    if (o < a.N) {
#pragma unroll
      for (int j = 0; j < NW / 8; ++j) {
        const int k = 8 * j + 2 * (lane & 3);
        if (k < a.K) part[(size_t)o * a.K + k] = d[4 * j + 2 * m] * inv;
        if (k + 1 < a.K) part[(size_t)o * a.K + k + 1] = d[4 * j + 2 * m + 1] * inv;
      }
    }
  }
  // bias: the 8 lanes of a column quad hold the 8 row groups
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], 1);
    bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], 2);
    bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], 4);
  }
  if (g == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (o0 + cy + i < a.N) a.part_b[(size_t)blockIdx.x * a.N + o0 + cy + i] = bsum[i];
  }
}

// dW[o, k] += sum_s part[s][o][k]  (s ascending),  db[o] += sum_s part_b[s][o]
__global__ void gw_wgrad_sum_kernel(const float* __restrict__ part, const float* __restrict__ part_b, int S, int N, int K, float* __restrict__ dW,
                                    int ldw, float* __restrict__ db) {
  const size_t nk = (size_t)N * K;
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < nk + N; e += (size_t)gridDim.x * blockDim.x) {
    if (e < nk) {
      float s = 0.f;
      for (int i = 0; i < S; ++i) s += part[(size_t)i * nk + e];
      dW[(e / K) * (size_t)ldw + e % K] += s;
    } else if (db) {
      const size_t o = e - nk;
      float s = 0.f;
      for (int i = 0; i < S; ++i) s += part_b[(size_t)i * N + o];
      db[o] += s;
    }
  }
}

// one CTA per SM over the (o block, row range) grid; row ranges hold whole chunks
static int splits_for(long long R, int gy) {
  const long long chunks = (R + RC - 1) / RC;
  long long s = GRID_SMS / gy;
  if (s < 1) s = 1;
  return (int)(chunks < s ? (chunks > 0 ? chunks : 1) : s);
}

}  // namespace wgt

namespace wgt {
// K > KB runs as blocks of KB columns of A (one kernel + sum pass each, in order, through the same partials)
constexpr int KB = 256;
}  // namespace wgt

size_t wgrad_tc_workspace_floats(long long R, int N, int K) {
  const int S = wgt::splits_for(R, (N + wgt::OB - 1) / wgt::OB);
  return (size_t)S * N * std::min(K, wgt::KB) + (size_t)S * N + 2;
}

cudaError_t launch_wgrad_tc(const float* dY, int ldy, int N, const RowSrc& a, int K, int rows_per_sample, int batch, float* dW, int ldw, float* db,
                            bool split, float* ws, size_t ws_floats, int32_t* status, cudaStream_t st) {
  using namespace wgt;
  if (N <= 0 || K <= 0 || rows_per_sample <= 0 || batch <= 0) return cudaErrorInvalidValue;
  if (a.kind != SRC_STREAM && a.kind != SRC_BCAST) return cudaErrorInvalidValue;
  const long long R = (long long)rows_per_sample * batch;
  const int gy = (N + OB - 1) / OB;
  const int S = splits_for(R, gy);
  if (ws_floats < wgrad_tc_workspace_floats(R, N, K)) return cudaErrorInvalidValue;
  Args g;
  g.dY = dY, g.ldy = ldy, g.N = N, g.a = a, g.rows = rows_per_sample, g.batch = batch, g.R = R;
  const long long chunks = (R + RC - 1) / RC;
  g.rows_per_cta = (int)(((chunks + S - 1) / S) * RC);
  g.part = ws, g.part_b = ws + (size_t)S * N * std::min(K, KB);
  float* amax = g.part_b + (size_t)S * N;
  g.amax = amax, g.status = status;
  cudaError_t e;
  if (split) {  // operand magnitudes (whole tensors: a valid bound for every row range)
    if ((e = cudaMemsetAsync(amax, 0, 2 * sizeof(float), st)) != cudaSuccess) return e;
    if ((e = launch_absmax_flat(dY, R * ldy, amax, st)) != cudaSuccess) return e;
    const long long arows = a.kind == SRC_BCAST ? rows_per_sample : (long long)batch * a.src_rows;
    if ((e = launch_absmax_flat(a.base, arows * a.ld, amax + 1, st)) != cudaSuccess) return e;
  }
  const dim3 grid(S, gy);
  for (int k0 = 0; k0 < K; k0 += KB) {  // dW[:, k0 .. k0 + kb) from A's columns k0 .. (the bias gradient with the first block)
    const int kb = std::min(KB, K - k0);
    g.K = kb, g.a = a, g.a.col0 = a.col0 + k0;
    const int nw = (kb + 63) / 64;  // 1..4
#define GW_WG(SPLIT_, NW_)                                                                                              \
    do {                                                                                                                \
      e = cudaFuncSetAttribute(gw_wgrad_tc_kernel<SPLIT_, NW_>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES); \
      if (e != cudaSuccess) return e;                                                                                   \
      gw_wgrad_tc_kernel<SPLIT_, NW_><<<grid, THREADS, SMEM_BYTES, st>>>(g);                                            \
    } while (0)
    if (split) {
      if (nw == 1) GW_WG(true, 64); else if (nw == 2) GW_WG(true, 128); else if (nw == 3) GW_WG(true, 192); else GW_WG(true, 256);
    } else {
      if (nw == 1) GW_WG(false, 64); else if (nw == 2) GW_WG(false, 128); else if (nw == 3) GW_WG(false, 192); else GW_WG(false, 256);
    }
#undef GW_WG
    count_launch();
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    gw_wgrad_sum_kernel<<<4 * GRID_SMS, 256, 0, st>>>(g.part, g.part_b, S, N, kb, dW + k0, ldw, k0 == 0 ? db : nullptr);
    count_launch();
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace gw
