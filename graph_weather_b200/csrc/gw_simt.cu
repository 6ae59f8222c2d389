// gw_simt.cu -- exact-fp32 row-op kernel on the CUDA cores (precision GW_PREC_FP32_SIMT).
//
// One kernel executes any gw::GemmOp: it assembles A rows from their row sources while staging them to shared
// memory (so the reference's cat / gather / scatter_sum intermediates never exist in HBM), runs an fp32 FFMA
// tile GEMM, and applies bias + gathered addends + ReLU + LayerNorm + residual in registers before one coalesced
// store.  It serves (a) every op of the forward when hidden sizes are not the 256 the wgmma kernel is built for,
// (b) the one-off weight-constant precompute, and (c) as the on-device fp32 cross-check of the tensor-core path.
//
// Tile: 64 rows x 256 cols per CTA (so a LayerNorm row never leaves the CTA), BK = 16, 256 threads; each thread
// owns 8 rows x 8 cols (cols strided by 32 so smem reads are conflict-free and global stores coalesce); a warp
// owns 8 complete rows, so LayerNorm statistics are 5 shuffles.
#include <cuda_runtime.h>

#include <algorithm>

#include "gw_ops.h"
#include "gw_internal.h"

namespace gw {

constexpr int BM = 64, BN = 256, BK = 16, NT = 256;

__device__ __forceinline__ float fetch_src(const RowSrc& s, int b, int i, int k) {
  switch (s.kind) {
    case SRC_STREAM:
      return __ldg(s.base + ((size_t)b * s.src_rows + i) * s.ld + s.col0 + k);
    case SRC_BCAST:
      return __ldg(s.base + (size_t)i * s.ld + s.col0 + k);
    case SRC_GATHER:
      return __ldg(s.base + ((size_t)b * s.src_rows + __ldg(s.idx + i)) * s.ld + s.col0 + k);
    case SRC_BGATHER:
      return __ldg(s.base + (size_t)__ldg(s.idx + i) * s.ld + s.col0 + k);
    case SRC_SEGSUM: {
      int j0 = __ldg(s.ptr + i), j1 = __ldg(s.ptr + i + 1);
      float acc = 0.f;
      for (int j = j0; j < j1; ++j) {  // same left-to-right order as scatter_add over the reference edge list
        int e = s.perm ? __ldg(s.perm + j) : j;
        acc += __ldg(s.base + ((size_t)b * s.src_rows + e) * s.ld + s.col0 + k);
      }
      return acc;
    }
    case SRC_GATHER_BCAST_RELU: {
      float v = __ldg(s.base + ((size_t)b * s.src_rows + __ldg(s.idx + i)) * s.ld + s.col0 + k) +
                __ldg(s.base2 + (size_t)i * s.ld2 + k);
      return v < 0.f ? 0.f : v;  // torch.relu: a NaN passes through (fmaxf would return 0)
    }
    default:
      return 0.f;
  }
}

__global__ void __launch_bounds__(NT) gw_rowop_f32_kernel(const GemmOp op) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Ws[BK][BN + 1];

  const int tid = threadIdx.x;
  const int tx = tid & 31, ty = tid >> 5;
  const int R = op.rows_per_sample * op.batch;
  const int row0 = blockIdx.x * BM;
  const int col0 = blockIdx.y * BN;
  const int K = op.K, N = op.N;
  const int k_split = op.a[0].width;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += BK) {
    // A tile: 64 x 16, element e -> (row e/16, k e%16): 16 consecutive lanes read 16 consecutive k of one row
#pragma unroll
    for (int it = 0; it < (BM * BK) / NT; ++it) {
      int e = tid + it * NT;
      int r = e / BK, kk = e % BK;
      int gr = row0 + r, gk = k0 + kk;
      float v = 0.f;
      if (gr < R && gk < K) {
        int b = gr / op.rows_per_sample, i = gr - b * op.rows_per_sample;
        v = (gk < k_split) ? fetch_src(op.a[0], b, i, gk) : fetch_src(op.a[1], b, i, gk - k_split);
      }
      As[kk][r] = v;
    }
    // W tile: 256 x 16 from W[n, k] (k contiguous)
#pragma unroll
    for (int it = 0; it < (BN * BK) / NT; ++it) {
      int e = tid + it * NT;
      int n = e / BK, kk = e % BK;
      int gn = col0 + n, gk = k0 + kk;
      Ws[kk][n] = (gn < N && gk < K) ? __ldg(op.W + (size_t)gn * op.ldw + gk) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[8], w[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = As[kk][ty * 8 + i];
#pragma unroll
      for (int j = 0; j < 8; ++j) w[j] = Ws[kk][tx + 32 * j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
    __syncthreads();
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gr = row0 + ty * 8 + i;
    const bool row_ok = gr < R;  // warp-uniform
    int b = 0, li = 0;
    if (row_ok) {
      b = gr / op.rows_per_sample;
      li = gr - b * op.rows_per_sample;
    }
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int gn = col0 + tx + 32 * j;
      float x = acc[i][j];
      if (row_ok && gn < N) {
        if (op.bias) x += __ldg(op.bias + gn);
#pragma unroll
        for (int s = 0; s < 3; ++s)
          if (op.add[s].kind != SRC_NONE) x += fetch_src(op.add[s], b, li, gn);
        if (op.relu) x = x < 0.f ? 0.f : x;  // torch.relu: NaN stays NaN, -0.0 stays -0.0
      } else {
        x = 0.f;
      }
      v[j] = x;
    }
    if (op.save_pre && row_ok) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int gn = col0 + tx + 32 * j;
        if (gn < N) op.save_pre[(size_t)gr * op.ldo + gn] = v[j];
      }
    }
    if (op.ln_gamma) {  // LayerNorm over N (<= 256, one CTA column block), eps = 1e-5, biased variance (torch)
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s / (float)N;
      float q = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int gn = col0 + tx + 32 * j;
        float d = (gn < N) ? v[j] - mean : 0.f;
        q += d * d;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = 1.0f / sqrtf(q / (float)N + 1e-5f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int gn = col0 + tx + 32 * j;
        if (gn < N) v[j] = (v[j] - mean) * rstd * __ldg(op.ln_gamma + gn) + __ldg(op.ln_beta + gn);
      }
    }
    if (row_ok) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int gn = col0 + tx + 32 * j;
        if (gn < N) {
          float x = v[j];
          if (op.residual.kind != SRC_NONE) x += fetch_src(op.residual, b, li, gn);
          // torch's threshold_backward: zero where mask <= 0, so a NaN mask entry lets the gradient through
          if (op.mask.kind != SRC_NONE && fetch_src(op.mask, b, li, gn) <= 0.f) x = 0.f;
          op.out[(size_t)gr * op.ldo + gn] = x;
        }
      }
    }
  }
}

// out[(b*rows + i), :] = sum over CSR segment i of base rows (left to right, the reference's scatter_add order).
// One 64-thread CTA per (segment, sample): float4 per thread across 256 columns, rows read fully coalesced.  Serves the
// encoder's lat/lon -> mesh aggregation, whose segments are very skewed (a polar cell collects thousands of points).
// VEC = false: one float per thread, for widths, strides or base pointers that float4 cannot address (an edge_dim of 30); each
// column is summed in the same order, so a width the float4 path also takes gives the same bits either way.
template <bool VEC>
__global__ void __launch_bounds__(64) gw_segsum_kernel(const float* __restrict__ base, int ld, int width,
                                                       const int32_t* __restrict__ ptr, const int32_t* __restrict__ perm,
                                                       int src_rows, int rows, float* __restrict__ out, int ldo, int ptr_base,
                                                       int accumulate) {
  const int i = blockIdx.x, b = blockIdx.y;
  const int j0 = __ldg(ptr + i) - ptr_base, j1 = __ldg(ptr + i + 1) - ptr_base;
  if (!VEC) {
    for (int c = threadIdx.x; c < width; c += 64) {
      float acc = 0.f;
      for (int j = j0; j < j1; ++j) {
        const int e = perm ? __ldg(perm + j) : j;
        acc += __ldg(base + ((size_t)b * src_rows + e) * ld + c);
      }
      float* o = out + ((size_t)b * rows + i) * ldo + c;
      *o = accumulate ? *o + acc : acc;
    }
    return;
  }
  for (int c = threadIdx.x * 4; c < width; c += 256) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = j0; j < j1; ++j) {
      const int e = perm ? __ldg(perm + j) : j;
      const float4 t = __ldg(reinterpret_cast<const float4*>(base + ((size_t)b * src_rows + e) * ld + c));
      acc.x += t.x, acc.y += t.y, acc.z += t.z, acc.w += t.w;
    }
    float4* o = reinterpret_cast<float4*>(out + ((size_t)b * rows + i) * ldo + c);
    if (accumulate) {  // the segment's sum is added to what an earlier call left (a sum split over row ranges)
      const float4 t = *o;
      acc.x = t.x + acc.x, acc.y = t.y + acc.y, acc.z = t.z + acc.z, acc.w = t.w + acc.w;
    }
    *o = acc;
  }
}

// float4 access to rows of stride ld from p: 16-byte aligned rows, whole float4 per row
static bool float4_rows(const void* p, int ld, int width) { return !(reinterpret_cast<uintptr_t>(p) & 15) && !(ld & 3) && !(width & 3); }

cudaError_t launch_segsum(const float* base, int ld, int width, const int32_t* ptr, const int32_t* perm, int src_rows,
                          int rows, int batch, float* out, int ldo, cudaStream_t stream, int ptr_base, bool accumulate) {
  if (rows <= 0 || batch <= 0) return cudaSuccess;
  if (float4_rows(base, ld, width) && float4_rows(out, ldo, width))
    gw_segsum_kernel<true><<<dim3(rows, batch), 64, 0, stream>>>(base, ld, width, ptr, perm, src_rows, rows, out, ldo, ptr_base, accumulate ? 1 : 0);
  else
    gw_segsum_kernel<false><<<dim3(rows, batch), 64, 0, stream>>>(base, ld, width, ptr, perm, src_rows, rows, out, ldo, ptr_base, accumulate ? 1 : 0);
  count_launch();
  return cudaGetLastError();
}

// ---- two-level segment sum for very uneven segments (the encoder: a polar mesh cell collects thousands of lat/lon points at
// 0.25 degree, most cells a few) ------------------------------------------------------------------------------------------
// Segments are cut into chunks of <= SEG_CHUNK rows (chunk table built on the device by gw_seg_chunks_kernel whenever the graph
// changes); one CTA sums one chunk with four independent row loads in flight; segments of one chunk are written straight to
// the output, longer ones leave per-chunk partial sums that gw_segsum_finish_kernel adds in chunk order.  Deterministic; the
// order differs from one long left-to-right sum only in where the partial sums are cut.
constexpr int SEG_CHUNK = 64;
// one block: every thread counts the chunks of a contiguous run of segments, a block-wide exclusive scan places them
__global__ void __launch_bounds__(1024) gw_seg_chunks_kernel(const int32_t* __restrict__ ptr, int n_seg, int32_t* __restrict__ chunk_seg,
                                                             int32_t* __restrict__ chunk_j0, int32_t* __restrict__ seg_chunk0) {
  __shared__ int warp_tot[32];
  const int t = threadIdx.x, ipt = (n_seg + 1023) / 1024;
  const int i0 = min(t * ipt, n_seg), i1 = min(i0 + ipt, n_seg);
  int mine = 0;
  for (int i = i0; i < i1; ++i) mine += max(1, (ptr[i + 1] - ptr[i] + SEG_CHUNK - 1) / SEG_CHUNK);  // empty segment: one empty chunk (zeroes its row)
  int incl = mine;
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if ((t & 31) >= o) incl += v;
  }
  if ((t & 31) == 31) warp_tot[t >> 5] = incl;
  __syncthreads();
  if (t < 32) {
    int w = warp_tot[t];
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, w, o);
      if (t >= o) w += v;
    }
    warp_tot[t] = w;
  }
  __syncthreads();
  int c = incl - mine + ((t >> 5) ? warp_tot[(t >> 5) - 1] : 0);
  for (int i = i0; i < i1; ++i) {
    seg_chunk0[i] = c;
    const int j0 = ptr[i], j1 = ptr[i + 1];
    int j = j0;
    do {
      chunk_seg[c] = i, chunk_j0[c] = j, ++c;
      j += SEG_CHUNK;
    } while (j < j1);
  }
  if (t == 1023) seg_chunk0[n_seg] = warp_tot[31];
}
__global__ void __launch_bounds__(64) gw_segsum_chunk_kernel(const float* __restrict__ base, int ld, const int32_t* __restrict__ ptr,
                                                             const int32_t* __restrict__ perm, int src_rows, int rows,
                                                             const int32_t* __restrict__ chunk_seg, const int32_t* __restrict__ chunk_j0,
                                                             const int32_t* __restrict__ seg_chunk0, int max_chunks, float* __restrict__ partial,
                                                             float* __restrict__ out, int ldo) {
  const int c = blockIdx.x, b = blockIdx.y;
  if (c >= __ldg(seg_chunk0 + rows)) return;
  const int seg = __ldg(chunk_seg + c), j0 = __ldg(chunk_j0 + c), j1 = min(j0 + SEG_CHUNK, __ldg(ptr + seg + 1));
  const float* src = base + (size_t)b * src_rows * ld + threadIdx.x * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int j = j0;
  for (; j + 4 <= j1; j += 4) {
    int e[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) e[u] = perm ? __ldg(perm + j + u) : j + u;
    float4 t[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) t[u] = __ldg(reinterpret_cast<const float4*>(src + (size_t)e[u] * ld));
#pragma unroll
    for (int u = 0; u < 4; ++u) acc.x += t[u].x, acc.y += t[u].y, acc.z += t[u].z, acc.w += t[u].w;
  }
  for (; j < j1; ++j) {
    const int e = perm ? __ldg(perm + j) : j;
    const float4 t = __ldg(reinterpret_cast<const float4*>(src + (size_t)e * ld));
    acc.x += t.x, acc.y += t.y, acc.z += t.z, acc.w += t.w;
  }
  const bool single = __ldg(seg_chunk0 + seg + 1) - __ldg(seg_chunk0 + seg) == 1;
  float* dst = single ? out + ((size_t)b * rows + seg) * ldo : partial + ((size_t)b * max_chunks + c) * 256;
  *reinterpret_cast<float4*>(dst + threadIdx.x * 4) = acc;
}
__global__ void __launch_bounds__(64) gw_segsum_finish_kernel(const float* __restrict__ partial, const int32_t* __restrict__ seg_chunk0, int rows,
                                                              int max_chunks, float* __restrict__ out, int ldo) {
  const int seg = blockIdx.x, b = blockIdx.y;
  const int c0 = __ldg(seg_chunk0 + seg), c1 = __ldg(seg_chunk0 + seg + 1);
  if (c1 - c0 <= 1) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = c0; c < c1; ++c) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(partial + ((size_t)b * max_chunks + c) * 256 + threadIdx.x * 4));
    acc.x += t.x, acc.y += t.y, acc.z += t.z, acc.w += t.w;
  }
  *reinterpret_cast<float4*>(out + ((size_t)b * rows + seg) * ldo + threadIdx.x * 4) = acc;
}
int seg_chunk_bound(int n_seg, int n_rows) { return n_seg + (n_rows + SEG_CHUNK - 1) / SEG_CHUNK + 1; }
cudaError_t launch_seg_chunks(const int32_t* ptr, int n_seg, int32_t* chunk_seg, int32_t* chunk_j0, int32_t* seg_chunk0, cudaStream_t st) {
  gw_seg_chunks_kernel<<<1, 1024, 0, st>>>(ptr, n_seg, chunk_seg, chunk_j0, seg_chunk0);
  count_launch();
  return cudaGetLastError();
}
// width must be 256 (one float4 per thread of the 64-thread CTA)
cudaError_t launch_segsum_chunked(const float* base, int ld, const int32_t* ptr, const int32_t* perm, int src_rows, int rows, int batch,
                                  const int32_t* chunk_seg, const int32_t* chunk_j0, const int32_t* seg_chunk0, int max_chunks, float* partial,
                                  float* out, int ldo, cudaStream_t st) {
  if (rows <= 0 || batch <= 0) return cudaSuccess;
  if ((ld & 3) || (ldo & 3)) return cudaErrorInvalidValue;
  gw_segsum_chunk_kernel<<<dim3(max_chunks, batch), 64, 0, st>>>(base, ld, ptr, perm, src_rows, rows, chunk_seg, chunk_j0, seg_chunk0, max_chunks,
                                                                partial, out, ldo);
  gw_segsum_finish_kernel<<<dim3(rows, batch), 64, 0, st>>>(partial, seg_chunk0, rows, max_chunks, out, ldo);
  count_launch(2);
  return cudaGetLastError();
}

// ---- backward primitives (exact fp32; gw_train.cu) --------------------------------------------------------------------------
// dW[n, k] += sum_r dY[r, n] * A[r, k]   (and db[n] += sum_r dY[r, n]) over R = rows_per_sample * batch rows, A assembled from a row
// source like the forward kernel does (N > 256: one launch per block of 256 outputs).  Tile: all N <= 256 output rows x 32
// k-columns per CTA column (blockIdx.y), the rows are
// cut into gridDim.x slabs; every CTA accumulates its slab in registers (8 n x 4 k per thread).  gw_wgrad_kernel adds it to dW
// with float atomics (summation order across slabs is not fixed: gradients repeat to ~1e-7 relative, not bit for bit);
// gw_wgrad_det_kernel stores it as slab blockIdx.x's partial tile, and gw_wgrad_sum_kernel adds the slabs in slab order.
constexpr int WG_KT = 32, WG_RT = 16;
template <bool PARTIAL>  // PARTIAL: store the slab's sums at dW / db (a partial tile) instead of adding them with atomics
__device__ __forceinline__ void wgrad_slab(const float* __restrict__ dY, int ldy, int N, RowSrc a, int K, int rows_per_sample, int batch,
                                           float* __restrict__ dW, int ldw, float* __restrict__ db) {
  __shared__ float Ys[WG_RT][256 + 1];
  __shared__ float As[WG_RT][WG_KT + 1];
  const int tid = threadIdx.x, tn = tid & 31, tk = tid >> 5;  // thread: n = tn + 32 i (i < 8), k = 4 tk + j (j < 4)
  const long long R = (long long)rows_per_sample * batch;
  const long long per = (R + gridDim.x - 1) / gridDim.x, r0 = blockIdx.x * per, r1 = min(R, r0 + per);
  const int k0 = blockIdx.y * WG_KT;
  float acc[8][4];
  float bacc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    bacc[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  }
  for (long long rb = r0; rb < r1; rb += WG_RT) {
    for (int e = tid; e < WG_RT * 256; e += 256) {
      const int r = e >> 8, n = e & 255;
      const long long gr = rb + r;
      Ys[r][n] = (gr < r1 && n < N) ? __ldg(dY + gr * ldy + n) : 0.f;
    }
    for (int e = tid; e < WG_RT * WG_KT; e += 256) {
      const int r = e / WG_KT, kk = e % WG_KT;
      const long long gr = rb + r;
      float v = 0.f;
      if (gr < r1 && k0 + kk < K) {
        const int b = (int)(gr / rows_per_sample), i = (int)(gr - (long long)b * rows_per_sample);
        v = fetch_src(a, b, i, k0 + kk);
      }
      As[r][kk] = v;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < WG_RT; ++r) {
      float y[8], x[4];
#pragma unroll
      for (int i = 0; i < 8; ++i) y[i] = Ys[r][tn + 32 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = As[r][4 * tk + j];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        bacc[i] += y[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(y[i], x[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int n = tn + 32 * i;
    if (n >= N) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + 4 * tk + j;
      if (k < K) {
        if (PARTIAL) dW[(size_t)n * ldw + k] = acc[i][j];
        else atomicAdd(dW + (size_t)n * ldw + k, acc[i][j]);
      }
    }
    if (db && blockIdx.y == 0 && tk == 0) {
      if (PARTIAL) db[n] = bacc[i];
      else atomicAdd(db + n, bacc[i]);
    }
  }
}
__global__ void __launch_bounds__(256) gw_wgrad_kernel(const float* __restrict__ dY, int ldy, int N, RowSrc a, int K, int rows_per_sample, int batch,
                                                       float* __restrict__ dW, int ldw, float* __restrict__ db) {
  wgrad_slab<false>(dY, ldy, N, a, K, rows_per_sample, batch, dW, ldw, db);
}
// part [gridDim.x][N][K], part_b [gridDim.x][N] (null: no bias): every element of slab blockIdx.x's tile is written
__global__ void __launch_bounds__(256) gw_wgrad_det_kernel(const float* __restrict__ dY, int ldy, int N, RowSrc a, int K, int rows_per_sample,
                                                           int batch, float* __restrict__ part, float* __restrict__ part_b) {
  wgrad_slab<true>(dY, ldy, N, a, K, rows_per_sample, batch, part + (size_t)blockIdx.x * N * K, K,
                   part_b ? part_b + (size_t)blockIdx.x * N : nullptr);
}
cudaError_t launch_wgrad(const float* dY, int ldy, int N, const RowSrc& a, int K, int rows_per_sample, int batch, float* dW, int ldw, float* db,
                         cudaStream_t st) {
  const long long R = (long long)rows_per_sample * batch;
  if (R <= 0 || N <= 0 || K <= 0) return cudaSuccess;
  const int slabs = (int)std::min<long long>(296, (R + 255) / 256);
  for (int o0 = 0; o0 < N; o0 += 256) {  // output blocks of 256 (the Ys tile), each a launch over all rows
    gw_wgrad_kernel<<<dim3(slabs, (K + WG_KT - 1) / WG_KT), 256, 0, st>>>(dY + o0, ldy, std::min(256, N - o0), a, K, rows_per_sample, batch,
                                                                           dW + (size_t)o0 * ldw, ldw, db ? db + o0 : nullptr);
    count_launch();
  }
  return cudaGetLastError();
}
// Slabs of the fixed-order weight gradient: those of launch_wgrad, fewer where the partial tiles of one output block of 256 would
// not fit in DET_WS_BYTES (train/run.py's 1024 x 1024 weights: 31 slabs).  From the shapes alone, so the summation order is too.
static int wgrad_det_slabs(long long R, int N, int K) {
  const size_t tile = (size_t)std::min(N, 256) * K + std::min(N, 256);
  const long long fit = (long long)(DET_WS_BYTES / sizeof(float) / tile);
  return (int)std::max(1LL, std::min({296LL, (R + 255) / 256, fit}));
}
size_t wgrad_det_workspace_floats(long long R, int N, int K) {
  if (R <= 0 || N <= 0 || K <= 0) return 0;
  return (size_t)wgrad_det_slabs(R, N, K) * ((size_t)std::min(N, 256) * K + std::min(N, 256));
}
cudaError_t launch_wgrad_det(const float* dY, int ldy, int N, const RowSrc& a, int K, int rows_per_sample, int batch, float* dW, int ldw, float* db,
                             float* ws, size_t ws_floats, cudaStream_t st) {
  const long long R = (long long)rows_per_sample * batch;
  if (R <= 0 || N <= 0 || K <= 0) return cudaSuccess;
  if (ws_floats < wgrad_det_workspace_floats(R, N, K)) return cudaErrorInvalidValue;
  const int slabs = wgrad_det_slabs(R, N, K);
  for (int o0 = 0; o0 < N; o0 += 256) {  // the output blocks one after the other through the same workspace
    const int nb = std::min(256, N - o0);
    float* part_b = db ? ws + (size_t)slabs * nb * K : nullptr;
    gw_wgrad_det_kernel<<<dim3(slabs, (K + WG_KT - 1) / WG_KT), 256, 0, st>>>(dY + o0, ldy, nb, a, K, rows_per_sample, batch, ws, part_b);
    count_launch();
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if ((e = launch_wgrad_sum(ws, part_b, slabs, nb, K, dW + (size_t)o0 * ldw, ldw, db ? db + o0 : nullptr, st)) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

// LayerNorm backward over rows of N <= 256 columns (one warp per row, rows grid-strided):
//   zh = (z - mean) * rstd;  g = dy * gamma;  dz = rstd * (g - mean(g) - zh * mean(g * zh));  dgamma += dy * zh;  dbeta += dy
// gw_ln_bwd_kernel adds each CTA's dgamma / dbeta sums with float atomics; gw_ln_bwd_det_kernel stores them as CTA blockIdx.x's
// partial rows (part [2][gridDim.x][N]: dgamma rows, then dbeta rows) and gw_colsum_kernel adds the CTAs in a fixed order.
template <bool PARTIAL>  // PARTIAL: store the CTA's sums at dgamma / dbeta (its partial rows) instead of adding them with atomics
__device__ __forceinline__ void ln_bwd_rows(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z, int ld_z, int N,
                                            const float* __restrict__ gamma, long long R, float* __restrict__ dz, int ld_dz,
                                            float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ float sg[8][256], sb[8][256];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float ag[8], ab[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) ag[j] = ab[j] = 0.f;
  for (long long r = (long long)blockIdx.x * 8 + w; r < R; r += (long long)gridDim.x * 8) {
    float zv[8], gv[8], dv[8];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = lane + 32 * j;
      zv[j] = c < N ? __ldg(z + r * ld_z + c) : 0.f;
      dv[j] = c < N ? __ldg(dy + r * ld_dy + c) : 0.f;
      s += zv[j];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)N;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = (lane + 32 * j < N) ? zv[j] - mean : 0.f;
      q += d * d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = 1.0f / sqrtf(q / (float)N + 1e-5f);
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = lane + 32 * j;
      const bool ok = c < N;
      zv[j] = ok ? (zv[j] - mean) * rstd : 0.f;
      gv[j] = ok ? dv[j] * __ldg(gamma + c) : 0.f;
      m1 += gv[j], m2 += gv[j] * zv[j];
      ag[j] += dv[j] * zv[j], ab[j] += dv[j];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m1 += __shfl_xor_sync(0xffffffffu, m1, o), m2 += __shfl_xor_sync(0xffffffffu, m2, o);
    m1 /= (float)N, m2 /= (float)N;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = lane + 32 * j;
      if (c < N) dz[r * ld_dz + c] = rstd * (gv[j] - m1 - zv[j] * m2);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) sg[w][lane + 32 * j] = ag[j], sb[w][lane + 32 * j] = ab[j];
  __syncthreads();
  const int c = threadIdx.x;
  if (c < N) {
    float g = 0.f, b = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) g += sg[k][c], b += sb[k][c];
    if (PARTIAL) dgamma[c] = g, dbeta[c] = b;
    else atomicAdd(dgamma + c, g), atomicAdd(dbeta + c, b);
  }
}
__global__ void __launch_bounds__(256) gw_ln_bwd_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z, int ld_z, int N,
                                                        const float* __restrict__ gamma, long long R, float* __restrict__ dz, int ld_dz,
                                                        float* __restrict__ dgamma, float* __restrict__ dbeta) {
  ln_bwd_rows<false>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, dgamma, dbeta);
}
__global__ void __launch_bounds__(256) gw_ln_bwd_det_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z, int ld_z, int N,
                                                            const float* __restrict__ gamma, long long R, float* __restrict__ dz, int ld_dz,
                                                            float* __restrict__ part) {
  ln_bwd_rows<true>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, part + (size_t)blockIdx.x * N, part + ((size_t)gridDim.x + blockIdx.x) * N);
}
// The same for rows of 256 < N <= 32 J columns (LN_BWD_MAX_N = 1024: the 1024-wide models of train/run.py:491-501): one warp per
// row with J values per lane (column lane + 32 j).  The per-CTA dgamma / dbeta partials of the 8 warps meet in one [8][1024]
// shared array, dgamma first, then dbeta (two [8][1024] arrays would not fit in 48 KB of static shared memory).
template <int J, bool PARTIAL>
__device__ __forceinline__ void ln_bwd_wide_rows(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z, int ld_z, int N,
                                                 const float* __restrict__ gamma, long long R, float* __restrict__ dz, int ld_dz,
                                                 float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ float sp[8][LN_BWD_MAX_N];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float ag[J], ab[J];
#pragma unroll
  for (int j = 0; j < J; ++j) ag[j] = ab[j] = 0.f;
  for (long long r = (long long)blockIdx.x * 8 + w; r < R; r += (long long)gridDim.x * 8) {
    float zv[J], dv[J];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int c = lane + 32 * j;
      zv[j] = c < N ? __ldg(z + r * ld_z + c) : 0.f;
      dv[j] = c < N ? __ldg(dy + r * ld_dy + c) : 0.f;
      s += zv[j];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)N;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const float d = (lane + 32 * j < N) ? zv[j] - mean : 0.f;
      q += d * d;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = 1.0f / sqrtf(q / (float)N + 1e-5f);
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int j = 0; j < J; ++j) {  // zv <- zh, dv <- g = dy * gamma (after the dgamma / dbeta terms have used dy)
      const int c = lane + 32 * j;
      const bool ok = c < N;
      zv[j] = ok ? (zv[j] - mean) * rstd : 0.f;
      ag[j] += dv[j] * zv[j], ab[j] += dv[j];
      dv[j] = ok ? dv[j] * __ldg(gamma + c) : 0.f;
      m1 += dv[j], m2 += dv[j] * zv[j];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m1 += __shfl_xor_sync(0xffffffffu, m1, o), m2 += __shfl_xor_sync(0xffffffffu, m2, o);
    m1 /= (float)N, m2 /= (float)N;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int c = lane + 32 * j;
      if (c < N) dz[r * ld_dz + c] = rstd * (dv[j] - m1 - zv[j] * m2);
    }
  }
#pragma unroll
  for (int j = 0; j < J; ++j)
    if (lane + 32 * j < N) sp[w][lane + 32 * j] = ag[j];
  __syncthreads();
  for (int c = threadIdx.x; c < N; c += 256) {
    float g = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) g += sp[k][c];
    if (PARTIAL) dgamma[c] = g;
    else atomicAdd(dgamma + c, g);
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < J; ++j)
    if (lane + 32 * j < N) sp[w][lane + 32 * j] = ab[j];
  __syncthreads();
  for (int c = threadIdx.x; c < N; c += 256) {
    float b = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) b += sp[k][c];
    if (PARTIAL) dbeta[c] = b;
    else atomicAdd(dbeta + c, b);
  }
}
template <int J>
__global__ void __launch_bounds__(256) gw_ln_bwd_wide_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z, int ld_z, int N,
                                                             const float* __restrict__ gamma, long long R, float* __restrict__ dz, int ld_dz,
                                                             float* __restrict__ dgamma, float* __restrict__ dbeta) {
  ln_bwd_wide_rows<J, false>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, dgamma, dbeta);
}
template <int J>
__global__ void __launch_bounds__(256) gw_ln_bwd_wide_det_kernel(const float* __restrict__ dy, int ld_dy, const float* __restrict__ z, int ld_z,
                                                                 int N, const float* __restrict__ gamma, long long R, float* __restrict__ dz,
                                                                 int ld_dz, float* __restrict__ part) {
  ln_bwd_wide_rows<J, true>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, part + (size_t)blockIdx.x * N,
                            part + ((size_t)gridDim.x + blockIdx.x) * N);
}
cudaError_t launch_ln_bwd(const float* dy, int ld_dy, const float* z, int ld_z, int N, const float* gamma, long long R, float* dz, int ld_dz,
                          float* dgamma, float* dbeta, cudaStream_t st) {
  if (R <= 0) return cudaSuccess;
  if (N > LN_BWD_MAX_N) return cudaErrorInvalidValue;
  const unsigned grid = (unsigned)std::min<long long>(GRID_SMS * 8, (R + 7) / 8);
  if (N <= 256)
    gw_ln_bwd_kernel<<<grid, 256, 0, st>>>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, dgamma, dbeta);
  else if (N <= 512)
    gw_ln_bwd_wide_kernel<16><<<grid, 256, 0, st>>>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, dgamma, dbeta);
  else
    gw_ln_bwd_wide_kernel<32><<<grid, 256, 0, st>>>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, dgamma, dbeta);
  count_launch();
  return cudaGetLastError();
}

// out0[c] += sum_s part[0][s][c],  out1[c] += sum_s part[1][s][c]  (s < S, c < N): thread row ty sums s = ty, ty + 32, ...
// ascending, then the 32 row sums are added in ty order -- an order fixed by S and N.
__global__ void __launch_bounds__(1024) gw_colsum_kernel(const float* __restrict__ part, int S, int N, float* __restrict__ out0,
                                                         float* __restrict__ out1) {
  __shared__ float sm[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5, c = blockIdx.x * 32 + tx;
  const float* p = part + (size_t)blockIdx.y * S * N;
  float acc = 0.f;
  if (c < N)
    for (int s = ty; s < S; s += 32) acc += __ldg(p + (size_t)s * N + c);
  sm[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && c < N) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) t += sm[k][tx];
    float* out = blockIdx.y ? out1 : out0;
    out[c] += t;
  }
}
size_t ln_bwd_det_workspace_floats(long long R, int N) {
  if (R <= 0 || N <= 0) return 0;
  return 2 * (size_t)std::min<long long>(GRID_SMS * 8, (R + 7) / 8) * N;
}
cudaError_t launch_ln_bwd_det(const float* dy, int ld_dy, const float* z, int ld_z, int N, const float* gamma, long long R, float* dz, int ld_dz,
                              float* dgamma, float* dbeta, float* ws, size_t ws_floats, cudaStream_t st) {
  if (R <= 0) return cudaSuccess;
  if (N > LN_BWD_MAX_N || ws_floats < ln_bwd_det_workspace_floats(R, N)) return cudaErrorInvalidValue;
  const unsigned grid = (unsigned)std::min<long long>(GRID_SMS * 8, (R + 7) / 8);  // the grid of launch_ln_bwd
  if (N <= 256)
    gw_ln_bwd_det_kernel<<<grid, 256, 0, st>>>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, ws);
  else if (N <= 512)
    gw_ln_bwd_wide_det_kernel<16><<<grid, 256, 0, st>>>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, ws);
  else
    gw_ln_bwd_wide_det_kernel<32><<<grid, 256, 0, st>>>(dy, ld_dy, z, ld_z, N, gamma, R, dz, ld_dz, ws);
  gw_colsum_kernel<<<dim3((N + 31) / 32, 2), 1024, 0, st>>>(ws, (int)grid, N, dgamma, dbeta);
  count_launch(2);
  return cudaGetLastError();
}

// out[i, c] (+)= sum_b in[(b * rows + i), c]     (gradient of a tensor that the forward broadcast over the batch)
__global__ void gw_batch_reduce_kernel(const float* __restrict__ in, int ld_in, long long rows, int width, int batch, float* __restrict__ out, int ld_out,
                                       int accumulate) {
  const long long total = rows * width;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / width;
    const int c = (int)(e - i * width);
    float s = accumulate ? out[i * ld_out + c] : 0.f;
    for (int b = 0; b < batch; ++b) s += __ldg(in + ((long long)b * rows + i) * ld_in + c);
    out[i * ld_out + c] = s;
  }
}
cudaError_t launch_batch_reduce(const float* in, int ld_in, long long rows, int width, int batch, float* out, int ld_out, bool accumulate,
                                cudaStream_t st) {
  if (rows <= 0 || width <= 0) return cudaSuccess;
  gw_batch_reduce_kernel<<<GRID_SMS * 4, 256, 0, st>>>(in, ld_in, rows, width, batch, out, ld_out, accumulate ? 1 : 0);
  count_launch();
  return cudaGetLastError();
}
// out[(b * rows + j), c] (+)= in[(b * src_rows + idx[j] - idx_base), c]   (gradient of a per-target sum: every row receives its target's
// gradient; idx_base: the first target of a table that holds a range of targets).  VEC: four columns per thread (float4), else one
// (any width, stride and alignment).
template <bool VEC>
__global__ void gw_gather_rows_kernel(const float* __restrict__ in, int ld_in, int src_rows, const int32_t* __restrict__ idx, long long rows, int width,
                                      int batch, float* __restrict__ out, int ld_out, int accumulate, int idx_base) {
  constexpr int V = VEC ? 4 : 1;
  const int q = width / V;
  const long long total = rows * batch * q;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long rj = e / q;
    const int c = (int)(e - rj * q) * V;
    const long long b = rj / rows, j = rj - b * rows;
    const float* src = in + (b * src_rows + (__ldg(idx + j) - idx_base)) * ld_in + c;
    float* dst = out + rj * ld_out + c;
    if (!VEC) {
      const float v = __ldg(src);
      *dst = accumulate ? *dst + v : v;
      continue;
    }
    const float4 v = __ldg(reinterpret_cast<const float4*>(src));
    float4* o = reinterpret_cast<float4*>(dst);
    if (accumulate) {
      float4 t = *o;
      t.x += v.x, t.y += v.y, t.z += v.z, t.w += v.w;
      *o = t;
    } else {
      *o = v;
    }
  }
}
cudaError_t launch_gather_rows(const float* in, int ld_in, int src_rows, const int32_t* idx, long long rows, int width, int batch, float* out,
                               int ld_out, bool accumulate, cudaStream_t st, int idx_base) {
  if (rows <= 0 || batch <= 0 || width <= 0) return cudaSuccess;
  if (float4_rows(in, ld_in, width) && float4_rows(out, ld_out, width))
    gw_gather_rows_kernel<true><<<GRID_SMS * 8, 256, 0, st>>>(in, ld_in, src_rows, idx, rows, width, batch, out, ld_out, accumulate ? 1 : 0, idx_base);
  else
    gw_gather_rows_kernel<false><<<GRID_SMS * 8, 256, 0, st>>>(in, ld_in, src_rows, idx, rows, width, batch, out, ld_out, accumulate ? 1 : 0, idx_base);
  count_launch();
  return cudaGetLastError();
}
// scatter = 0: out[(b * rows + j), c] = in[(b * other_rows + idx[j]), c]     (rows of a caller tensor picked through a permutation)
// scatter = 1: out[(b * other_rows + idx[j]), c] = in[(b * rows + j), c]     (and written back through it)
// Any width and stride (the 102 or 621 input features): one float per thread, 64-bit offsets throughout.
__global__ void gw_permute_rows_kernel(const float* __restrict__ in, int ld_in, const int32_t* __restrict__ idx, long long rows, int other_rows,
                                       int width, int batch, float* __restrict__ out, int ld_out, int scatter) {
  const long long total = rows * batch * width;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long rj = e / width;
    const int c = (int)(e - rj * width);
    const long long b = rj / rows, j = rj - b * rows;
    const long long far = b * other_rows + __ldg(idx + j);
    if (scatter)
      out[far * ld_out + c] = __ldg(in + rj * ld_in + c);
    else
      out[rj * ld_out + c] = __ldg(in + far * ld_in + c);
  }
}
cudaError_t launch_permute_rows(const float* in, int ld_in, const int32_t* idx, long long rows, int other_rows, int width, int batch, float* out,
                                int ld_out, bool scatter, cudaStream_t st) {
  if (rows <= 0 || batch <= 0 || width <= 0) return cudaSuccess;
  gw_permute_rows_kernel<<<GRID_SMS * 8, 256, 0, st>>>(in, ld_in, idx, rows, other_rows, width, batch, out, ld_out, scatter ? 1 : 0);
  count_launch();
  return cudaGetLastError();
}
// dst[r, c] += src[r, c] for c < width (rows of different strides)
__global__ void gw_strided_add_kernel(const float* __restrict__ src, int ld_src, float* __restrict__ dst, int ld_dst, long long rows, int width) {
  const long long total = rows * width;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / width;
    const int c = (int)(e - r * width);
    dst[r * ld_dst + c] += __ldg(src + r * ld_src + c);
  }
}
cudaError_t launch_strided_add(const float* src, int ld_src, float* dst, int ld_dst, long long rows, int width, cudaStream_t st) {
  if (rows <= 0 || width <= 0) return cudaSuccess;
  gw_strided_add_kernel<<<GRID_SMS * 4, 256, 0, st>>>(src, ld_src, dst, ld_dst, rows, width);
  count_launch();
  return cudaGetLastError();
}
// WT[k, n] = W[n, k]   (data gradients multiply by the untransposed weight: the row-op kernel wants it as [out-of-op, in-of-op])
__global__ void gw_transpose_kernel(const float* __restrict__ W, int rows, int cols, float* __restrict__ WT) {
  __shared__ float t[32][33];
  const int x = blockIdx.x * 32 + threadIdx.x, y0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8)
    if (x < cols && y0 + j < rows) t[j][threadIdx.x] = W[(size_t)(y0 + j) * cols + x];
  __syncthreads();
  const int xo = blockIdx.y * 32 + threadIdx.x, yo0 = blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += 8)
    if (xo < rows && yo0 + j < cols) WT[(size_t)(yo0 + j) * rows + xo] = t[threadIdx.x][j];
}
cudaError_t launch_transpose(const float* W, int rows, int cols, float* WT, cudaStream_t st) {
  gw_transpose_kernel<<<dim3((cols + 31) / 32, (rows + 31) / 32), dim3(32, 8), 0, st>>>(W, rows, cols, WT);
  count_launch();
  return cudaGetLastError();
}

// running max |x| for a magnitude bound: a NaN becomes +inf and stays (fmaxf would drop it and leave the bound finite)
__device__ __forceinline__ float amax1(float m, float x) {
  const float a = fabsf(x);
  return a <= m ? m : (a == a ? a : __int_as_float(0x7f800000));
}
__device__ __forceinline__ float amax4(float m, float4 v) { return amax1(amax1(amax1(amax1(m, v.x), v.y), v.z), v.w); }

// dst[r, 0:ld_dst] = [src[r, 0:width], 0 ...]: widens rows whose width / stride are not multiples of 64 floats (the 102
// input features) so that the tensor-core chain can read them with aligned 128-bit loads.  The pass sees every input value,
// so it also produces their absolute maximum (amax, may be null): the magnitude bound the chain's operand scaling starts from.
__global__ void __launch_bounds__(256) gw_pad_rows_kernel(const float* __restrict__ src, int ld_src, int width, float* __restrict__ dst,
                                                          int ld_dst, long long rows, float* __restrict__ amax) {
  const int q = ld_dst >> 2;  // float4 per destination row
  const long long total = rows * q;
  float m = 0.f;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / q;
    const int c = (int)(e - r * q) * 4;
    const float* s = src + r * ld_src + c;
    float4 v;
    v.x = (c + 0 < width) ? __ldg(s + 0) : 0.f;
    v.y = (c + 1 < width) ? __ldg(s + 1) : 0.f;
    v.z = (c + 2 < width) ? __ldg(s + 2) : 0.f;
    v.w = (c + 3 < width) ? __ldg(s + 3) : 0.f;
    m = amax4(m, v);
    *reinterpret_cast<float4*>(dst + r * ld_dst + c) = v;
  }
  if (amax) {
    if (!(m <= 3.0e38f)) m = __int_as_float(0x7f800000);  // NaN / inf inputs: the bound is infinite (the chain flags it)
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));  // m >= 0: int order == float order
  }
}
cudaError_t launch_pad_rows(const float* src, int ld_src, int width, float* dst, int ld_dst, long long rows, float* amax, cudaStream_t stream) {
  if (rows <= 0) return cudaSuccess;
  if (ld_dst & 3) return cudaErrorInvalidValue;
  gw_pad_rows_kernel<<<GRID_SMS * 8, 256, 0, stream>>>(src, ld_src, width, dst, ld_dst, rows, amax);
  count_launch();
  return cudaGetLastError();
}

// *amax = max(*amax, max |p[0..n)|) over a contiguous array (raw caller tensors entering a tensor-core chain).
__global__ void __launch_bounds__(256) gw_absmax_flat_kernel(const float* __restrict__ p, long long n, float* __restrict__ amax) {
  float m = 0.f;
  const long long head = min(n, (long long)((16 - (reinterpret_cast<uintptr_t>(p) & 15)) & 15) >> 2);
  const long long nv = (n - head) >> 2;
  const float4* pv = reinterpret_cast<const float4*>(p + head);
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < nv; e += (long long)gridDim.x * blockDim.x) {
    m = amax4(m, __ldg(pv + e));
  }
  if (blockIdx.x == 0 && threadIdx.x < 8) {  // unaligned head and tail
    for (long long e = threadIdx.x; e < head; e += 8) m = amax1(m, p[e]);
    for (long long e = head + 4 * nv + threadIdx.x; e < n; e += 8) m = amax1(m, p[e]);
  }
  if (!(m <= 3.0e38f)) m = __int_as_float(0x7f800000);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));
}
cudaError_t launch_absmax_flat(const float* p, long long n, float* amax, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  gw_absmax_flat_kernel<<<GRID_SMS * 4, 256, 0, stream>>>(p, n, amax);
  count_launch();
  return cudaGetLastError();
}

// ---- helpers of the fused per-target sums (gw_tc3.cu, F_SEG) ------------------------------------------------------------------
// stats[0] = longest CSR segment, stats[1] = shortest (caller initialises {0, INT_MAX}); dst[j] = i for ptr[i] <= j < ptr[i+1]
__global__ void gw_csr_expand_kernel(const int32_t* __restrict__ ptr, int n, int32_t* __restrict__ dst, int* __restrict__ stats) {
  int mx = 0, mn = 0x7fffffff;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int j0 = ptr[i], j1 = ptr[i + 1];
    mx = max(mx, j1 - j0), mn = min(mn, j1 - j0);
    if (dst)
      for (int j = j0; j < j1; ++j) dst[j] = i;
  }
  for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o)), mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  if ((threadIdx.x & 31) == 0) atomicMax(stats, mx), atomicMin(stats + 1, mn);
}
cudaError_t launch_csr_expand(const int32_t* ptr, int n, int32_t* dst, int* stats, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  gw_csr_expand_kernel<<<(n + 255) / 256 < 1184 ? (n + 255) / 256 : 1184, 256, 0, stream>>>(ptr, n, dst, stats);
  count_launch();
  return cudaGetLastError();
}
// A segment cut by a 16-row group boundary of the chain kernel's tiles (the rows one worker warp reduces, gw_tc3.cu) left the
// sum of its later rows in `carry` ([batch][tiles][8][256]); add it to the segment's row of out.  64 threads per boundary, four
// boundaries per CTA (a quarter of a million one-boundary CTAs cost more in launch overhead than in work); fixed order.
__global__ void __launch_bounds__(256) gw_seg_carry_kernel(const float* __restrict__ carry, const int32_t* __restrict__ seg_dst, int rows,
                                                           int tiles, int seg_rows, float* __restrict__ out, int ldo) {
  const int bg = blockIdx.x * 4 + (threadIdx.x >> 6), b = blockIdx.y;  // boundary = tile * 8 + group
  const int t = threadIdx.x & 63;
  if (bg >= tiles * 8) return;
  const int r = (bg >> 3) * 128 + (bg & 7) * 16;
  if (r <= 0 || r >= rows) return;
  const int d = __ldg(seg_dst + r);
  if (__ldg(seg_dst + r - 1) != d) return;  // the group starts a new segment: nothing was carried
  const float4 c = __ldg(reinterpret_cast<const float4*>(carry + ((size_t)b * tiles * 8 + bg) * 256 + t * 4));
  float4* o = reinterpret_cast<float4*>(out + ((size_t)b * seg_rows + d) * (size_t)ldo + t * 4);
  float4 v = *o;
  v.x += c.x, v.y += c.y, v.z += c.z, v.w += c.w;
  *o = v;
}
cudaError_t launch_seg_carry(const float* carry, const int32_t* seg_dst, int rows, int seg_rows, int batch, float* out, int ldo,
                             cudaStream_t stream) {
  if (rows <= 0 || batch <= 0) return cudaSuccess;
  const int tiles = (rows + 127) / 128;
  gw_seg_carry_kernel<<<dim3(tiles * 2, batch), 256, 0, stream>>>(carry, seg_dst, rows, tiles, seg_rows, out, ldo);
  count_launch();
  return cudaGetLastError();
}

// Rows wider than one CTA column block (N > 256, e.g. the 1024-wide models of train/run.py:491-501): the row op above runs
// without its LayerNorm / residual and this kernel finishes the rows in place: out = residual + LN(out).  One warp per row,
// two passes over the (L2-resident) row like torch's LayerNorm (mean, then biased variance, eps 1e-5).  The tensor-core row ops
// of a layer-by-layer plan (gw_forward.cu, tc_row_op) finish their LayerNorm'd rows here too; amax (optional, zeroed by the
// caller: a tensor written in chunks accumulates) then takes max |out| of the rows written, the bound the next layer's fp16 hi/lo split is scaled from (infinite when a
// row is not finite).
__global__ void __launch_bounds__(256) gw_ln_rows_kernel(const GemmOp op, float* __restrict__ amax) {
  const int lane = threadIdx.x & 31;
  const long long R = (long long)op.rows_per_sample * op.batch;
  const long long gr = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (gr >= R) return;
  const int b = (int)(gr / op.rows_per_sample), li = (int)(gr - (long long)b * op.rows_per_sample);
  float* row = op.out + (size_t)gr * op.ldo;
  const int N = op.N;
  float s = 0.f;
  for (int c = lane; c < N; c += 32) s += row[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)N;
  float q = 0.f;
  for (int c = lane; c < N; c += 32) {
    const float d = row[c] - mean;
    q += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = 1.0f / sqrtf(q / (float)N + 1e-5f);
  float m = 0.f;
  for (int c = lane; c < N; c += 32) {
    float x = (row[c] - mean) * rstd * __ldg(op.ln_gamma + c) + __ldg(op.ln_beta + c);
    if (op.residual.kind != SRC_NONE) x += fetch_src(op.residual, b, li, c);
    row[c] = x;
    m = amax1(m, x);
  }
  if (amax) {
    if (!(m <= 3.0e38f)) m = __int_as_float(0x7f800000);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) atomicMax(reinterpret_cast<int*>(amax), __float_as_int(m));  // m >= 0: int order == float order
  }
}
cudaError_t launch_ln_rows(const GemmOp& op, float* amax, cudaStream_t stream) {
  const long long R = (long long)op.rows_per_sample * op.batch;
  if (R <= 0 || op.N <= 0) return cudaSuccess;
  gw_ln_rows_kernel<<<(unsigned)((R + 7) / 8), 256, 0, stream>>>(op, amax);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_rowop_simt(const GemmOp& op, cudaStream_t stream) {
  const long long R = (long long)op.rows_per_sample * op.batch;
  if (R <= 0 || op.N <= 0) return cudaSuccess;
  dim3 grid((unsigned)((R + BM - 1) / BM), (unsigned)((op.N + BN - 1) / BN));
  if (op.ln_gamma && op.N > BN) {
    GemmOp g = op;  // GEMM + bias + addends + ReLU only; LayerNorm and residual in the second kernel
    g.ln_gamma = g.ln_beta = nullptr;
    g.residual = RowSrc();
    gw_rowop_f32_kernel<<<grid, NT, 0, stream>>>(g);
    gw_ln_rows_kernel<<<(unsigned)((R + 7) / 8), 256, 0, stream>>>(op, nullptr);
    count_launch(2);
    return cudaGetLastError();
  }
  gw_rowop_f32_kernel<<<grid, NT, 0, stream>>>(op);
  count_launch();
  return cudaGetLastError();
}

}  // namespace gw
