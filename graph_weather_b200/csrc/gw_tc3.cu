// gw_tc3.cu -- the fused MLP-chain kernel on Hopper tensor cores (wgmma, fp32 accumulation in registers), precision
// GW_PREC_FP32_TC / BF16_TC.
//
// One persistent CTA per SM walks 128-row tiles of a gw::TcChain.  For every tile the whole chain
//     A0 = assemble(row sources)                                   (stream / gather / relu(gather+const) ...)
//     for each layer:  D = A . W^T  (wgmma.mma_async, fp32 accumulate in registers)
//                      v = D*s + bias + gathered addends ; ReLU | LayerNorm ; + residual
//                      v -> global (fp32)  and/or  v -> split fp16 hi/lo -> shared memory = A operand of the next layer
// runs without the activations ever leaving the SM: the reference's x[row]/x[col] gathers, cat, 3 Linear + LayerNorm and
// residual (graph_net_block.py:131-135, 184-191) are one kernel per edge pass and one per node pass.
//
// fp32 fidelity on fp16 tensor cores: every fp32 operand a is split a = hi + lo (two fp16, 22 significand bits) and each
// product is hi*hi + lo*hi + hi*lo with fp32 accumulation.  Weights are pre-scaled by a power of two so their lo parts stay
// normal; the scale is undone exactly in the epilogue.
//
// Layout of the work:
//   * two consumer warpgroups.  Warpgroup w owns the tile rows 64 w .. 64 w + 63 for the whole chain: it assembles their stage-0
//     operand, issues the m64nNk16 wgmma of every layer over them and runs each layer's epilogue on its own accumulator registers
//     (a 64 x 256 fp32 accumulator is 128 registers per thread).  A warpgroup writes and reads only its own operand rows, so the
//     two warpgroups share nothing but the weight stream.
//   * the wgmma accumulator gives lane t of warp q the rows 16 q + t/4 (+ 8) and, in every 8 columns, the pair 2 (t%4) + {0,1}.
//     The weights are packed with output rows and K columns permuted inside groups of 32 (perm32, gw_pack.cu) so that in every
//     32-column step a thread holds EIGHT CONSECUTIVE features of two rows: gathered addends / residual rows are loaded and
//     outputs stored directly from/to global memory with pairs of 128-bit accesses (four adjacent lanes cover one 128-byte line), no
//     staging.  Tile rows are handed out so that a thread's two rows are CONSECUTIVE logical rows (fr0, fr0 + 1 <-> operand rows
//     16 q + t/4 and + 8): the last layer of an edge chain reduces its rows per target node in registers and shuffles
//     (graph_net_block.py:188 scatter_sum, edges are target-sorted, segments of <= 8 rows) and stores per-node sums.
//   * the A operand lives in four 64-column slots ([128 x 64] hi|lo, 128 KB); a stage-0 operand wider than 256 columns is
//     assembled and multiplied in windows of four slots.  The result of a layer overwrites its own operand once that layer's
//     wgmma have completed.
//   * two instantiations per precision: the lean path (every source / output 32-byte aligned and as wide as the layer; the
//     epilogue is specialised per feature mask and fully unrolled) and the general path (any width / alignment).
//   * warp 8: weight producer (cp.async.bulk of pre-swizzled panels of up to 32 KB, two stages).  setmaxnreg gives the
//     consumers 240 registers and the producer warpgroup 24.
//   * operand range: every tensor carries a rigorous magnitude bound (device float); each CTA derives, per layer, the power
//     of two that brings the next fp16-split operand into [2^14, 2^15) and folds its inverse into the accumulator scale, so raw
//     (unnormalised) inputs cannot overflow fp16 and small ones keep normal lo parts.  The amax status bit stays as a guard.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "gw_internal.h"
#include "gw_ops.h"
#include "gw_tc_ptx.cuh"

namespace gw {
namespace t3 {

#ifdef GW_ABLATE
#define ABL3(bit) ((ch.ablate & (bit)) != 0)
#else
#define ABL3(bit) false
#endif
// the consumer's helpers are lambdas over the kernel's state: inlined, so that the accumulator array stays in registers
#define GW_INLINE __attribute__((always_inline))
enum { ABL_FENCE = 1, ABL_LOADS = 2, ABL_CONVERT = 4, ABL_STORES = 8, ABL_LN = 16, ABL_WEIGHTS = 128 };

// epilogue feature mask of a layer (TcLayer::kind); the lean path is instantiated for the masks that occur
enum { F_ADD0 = 1, F_ADD1 = 2, F_RELU = 4, F_LN = 8, F_RES = 16, F_OUT = 32, F_FEEDS = 64, F_SEG = 128, F_NARROW = 256 };
constexpr int TILE_M = 128;
constexpr int A_SLOTS = 4, B_STAGES = 2;
constexpr int A_HALF_BYTES = TILE_M * 128;      // [128 rows x 64 halfs]
constexpr int A_SLOT_BYTES = 2 * A_HALF_BYTES;  // hi | lo
constexpr int B_STAGE_BYTES = 256 * 128;        // [256 rows x 64 halfs], hi OR lo panel
constexpr int CONSUMERS = 2;                    // warpgroups, 64 tile rows each
constexpr int CONSUMER_WARPS = 4 * CONSUMERS, NUM_WORKERS = 32 * CONSUMER_WARPS;
constexpr int WARP_PRODUCER = CONSUMER_WARPS;
constexpr int NUM_THREADS = NUM_WORKERS + 128;  // + one producer warpgroup (one active warp)
constexpr int WORKER_REGS = 240, AUX_REGS = 24;  // 256 x 240 + 128 x 24 = 384 x 168: the launch allocation of __launch_bounds__(384, 1)
constexpr int PAR_LAYERS = 6;
constexpr int OFF_A = 0;
constexpr int OFF_B = A_SLOTS * A_SLOT_BYTES;
constexpr int OFF_BAR = OFF_B + B_STAGES * B_STAGE_BYTES;
constexpr int NUM_BARS = 2 * B_STAGES;
constexpr int OFF_PAR = OFF_BAR + 2 * NUM_BARS * 8;   // float bias[PAR_LAYERS][256]
constexpr int OFF_LNP = OFF_PAR + PAR_LAYERS * 1024;  // float gamma_beta[2][2][256]
constexpr int OFF_SCL = OFF_LNP + 4 * 1024;           // float scl[2 * PAR_LAYERS + 4]: per layer {accumulator scale, operand scale of the result}, then the stage-0 operand scale
constexpr int SMEM_BYTES = OFF_SCL + (2 * PAR_LAYERS + 4) * 4;
static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB per-CTA shared memory limit");
static_assert(OFF_B % 1024 == 0 && A_SLOT_BYTES % 1024 == 0 && B_STAGE_BYTES % 1024 == 0, "SWIZZLE_128B needs 1 KB alignment");

template <int I, int N, class Fn>
__device__ __forceinline__ void static_for(Fn&& f) {
  if constexpr (I < N) {
    f(std::integral_constant<int, I>{});
    static_for<I + 1, N>(f);
  }
}
template <int V>
using ic = std::integral_constant<int, V>;

__device__ __forceinline__ bool src_gathered(int kind) { return kind == SRC_GATHER || kind == SRC_BGATHER || kind == SRC_GATHER_BCAST_RELU; }
__device__ __forceinline__ bool src_per_sample(int kind) { return kind == SRC_STREAM || kind == SRC_GATHER || kind == SRC_GATHER_BCAST_RELU; }
__device__ __forceinline__ const char* src_sample_base(const RowSrc& s, int b) {
  return reinterpret_cast<const char*>(s.base + (src_per_sample(s.kind) ? (size_t)b * (size_t)s.src_rows * (size_t)s.ld : (size_t)0) + s.col0);
}
// my two row pointers into a source: tile rows i0 + rl[m] (through the index for gathered sources), first column cofs
__device__ __forceinline__ void row_ptrs2(const RowSrc& s, int b, int i0, const int (&rl)[2], int cofs, const char* (&p)[2]) {
  const char* base = src_sample_base(s, b) + 4 * cofs;
  const size_t ldb = 4 * (size_t)s.ld;
  if (src_gathered(s.kind)) {
#pragma unroll
    for (int k = 0; k < 2; ++k) p[k] = base + (size_t)(uint32_t)__ldg(s.idx + i0 + rl[k]) * ldb;
  } else {
#pragma unroll
    for (int k = 0; k < 2; ++k) p[k] = base + (size_t)(uint32_t)(i0 + rl[k]) * ldb;
  }
}
// 8 consecutive floats (32-byte aligned) in two 128-bit accesses: four adjacent lanes cover one full 128-byte line
__device__ __forceinline__ void ld256(const char* p, float* o) {
  asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%8];\n\t"
               "ld.global.nc.v4.f32 {%4, %5, %6, %7}, [%8+16];"
               : "=f"(o[0]), "=f"(o[1]), "=f"(o[2]), "=f"(o[3]), "=f"(o[4]), "=f"(o[5]), "=f"(o[6]), "=f"(o[7])
               : "l"(p));
}
__device__ __forceinline__ void st256(char* p, float a, float b, float c, float d, float e, float f, float g, float h) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};\n\t"
               "st.global.v4.f32 [%0+16], {%5, %6, %7, %8};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d), "f"(e), "f"(f), "f"(g), "f"(h)
               : "memory");
}
// General path: logical columns col .. col+7 of one row (zero at and beyond `width`), widest access the row's alignment allows
__device__ __forceinline__ void load8(const float* rowp, int col, int width, float* o) {
  const float* p = rowp + col;
  if (col + 8 <= width && (reinterpret_cast<uintptr_t>(p) & 31) == 0) {
    ld256(reinterpret_cast<const char*>(p), o);
  } else if (col + 8 <= width && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p + 4));
    o[0] = a.x, o[1] = a.y, o[2] = a.z, o[3] = a.w, o[4] = b.x, o[5] = b.y, o[6] = b.z, o[7] = b.w;
  } else {
#pragma unroll
    for (int t = 0; t < 8; ++t) o[t] = (col + t < width) ? __ldg(p + t) : 0.f;
  }
}
// row `r` (a tile row, clamped) of a source, as a float pointer at its first column (general path)
__device__ __forceinline__ const float* src_row(const RowSrc& s, int b, int i0, int r) {
  const int i = src_gathered(s.kind) ? __ldg(s.idx + i0 + r) : i0 + r;
  return reinterpret_cast<const float*>(src_sample_base(s, b)) + (size_t)(uint32_t)i * (size_t)s.ld;
}
// Fragment of one 32-column step (16 accumulator registers, 16 u .. 16 u + 15): index 4 g + 2 m + e = (row m of my two,
// feature 2 g + e of my eight).  FR(m, t): fragment index of (row m, feature t); PX(i): row-order index 8 m + t of fragment index i.
__host__ __device__ constexpr int FR(int m, int t) { return 4 * (t >> 1) + 2 * m + (t & 1); }
__host__ __device__ constexpr int PX(int i) { return 8 * ((i >> 1) & 1) + 2 * (i >> 2) + (i & 1); }
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
// column parameter (bias / LayerNorm gamma, beta: my 8 features as two float4) of fragment index i
__device__ __forceinline__ float col8(const float4& lo, const float4& hi, int i) {
  const int c = 2 * (i >> 2) + (i & 1);
  const float4& b = (c & 4) ? hi : lo;
  return (c & 2) ? ((c & 1) ? b.w : b.z) : ((c & 1) ? b.y : b.x);
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
// Operand store of one step.  Value (row m, feature t = 2 g + e of my eight) is accumulator column 32 fc + 8 g + 2 (lane % 4) + e of
// the 64-column chunk: half2 (e = 0, 1) at byte 4 (lane % 4) of 16-byte chunk 4 fc + g, swizzled with the operand row's low bits
// (= lane / 4).  `sa` = shared address of (my first row, g = 0) inside the slot: g flips bits 4-5, my second row is 8 operand
// rows (1 KB) further.  ROWORDER: v is in row order (stage 0) instead of fragment order (epilogues).
template <bool SPLIT, bool ROWORDER>
__device__ __forceinline__ void store_operand_x4(uint32_t sa, const float (&v)[16], float& amax) {
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int i = ROWORDER ? 8 * m + 2 * g : 4 * g + 2 * m;
      const float a0 = v[i], a1 = v[i + 1];
      amax = fmaxf(amax, fmaxf(fabsf(a0), fabsf(a1)));
      const uint32_t addr = (sa ^ (uint32_t)(g << 4)) + 1024u * m;
      if (SPLIT) {
        const __half2 hh = __floats2half2_rn(a0, a1);
        const float2 hf = __half22float2(hh);
        const __half2 ll = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
        sts32(addr, *reinterpret_cast<const uint32_t*>(&hh));
        sts32(addr + A_HALF_BYTES, *reinterpret_cast<const uint32_t*>(&ll));
      } else {
        const __nv_bfloat162 bb = __floats2bfloat162_rn(a0, a1);
        sts32(addr, *reinterpret_cast<const uint32_t*>(&bb));
      }
    }
}

// ---- operand range --------------------------------------------------------------------------------------------------
// The power of two s that brings a tensor bounded by m into [2^14, 2^15), up as well as down: large tensors stay under the fp16
// maximum (65504), and small ones (gradients ~1e-8, inputs in small physical units) keep normal fp16 lo parts.  The bound is
// rigorous, so scaling up cannot overflow.  1 when the bound is unknown (0) or not finite.
__device__ __forceinline__ float fit_scale(float m) {
  if (!(m > 0.f) || !(m < 3.0e38f)) return 1.f;
  int e = (int)((__float_as_uint(m) >> 23) & 0xffu) - 127;  // floor(log2 m) (normals)
  e = e < -110 ? -110 : e;
  return __uint_as_float((uint32_t)(127 + 14 - e) << 23);   // 2^(14-e)
}
__device__ __forceinline__ float ldbound(const float* p) { return p ? __ldg(p) : 0.f; }
__device__ __forceinline__ float srcbound(const RowSrc& s) {
  if (!s.bound) return 0.f;
  const float m = __ldg(s.bound) * s.bound_mul;
  return s.bound_mul_i ? m * (float)max(__ldg(s.bound_mul_i), 1) : m;
}

// ---- the product ------------------------------------------------------------------------------------------------------
// D (+)= A[:, 64 kc0 .. 64 kc1) . W^T over my warpgroup's 64 rows (a_rows): per 64-column chunk one weight panel (bf16) or two
// (fp16 hi, lo), four k16 steps each; A_hi.B_hi + A_lo.B_hi on the hi panel, A_hi.B_lo on the lo panel.  Everything here is
// warpgroup-uniform straight-line code (the waits loop inside their asm statements), so ptxas keeps the wgmma asynchronous.  A
// panel's stage is released by every consumer thread once the wgmma that read it have completed; the next panel is already
// resident (two stages), so the tensor pipe only idles for the issue latency between panels.
template <bool SPLIT, int N>
__device__ __forceinline__ void mma_chunks(float (&d)[128], uint32_t a_rows, uint32_t b_base, uint32_t bar_full_b, uint32_t bar_empty_b,
                                           uint32_t& bi, int kc0, int kc1) {
  for (int kc = kc0; kc < kc1; ++kc) {
    const uint32_t a_hi = a_rows + (uint32_t)(kc % A_SLOTS) * A_SLOT_BYTES, a_lo = a_hi + A_HALF_BYTES;
#pragma unroll
    for (int part = 0; part < (SPLIT ? 2 : 1); ++part) {
      const uint32_t stage = bi % B_STAGES, nb = bi / B_STAGES;
      mbar_wait_or_trap(bar_full_b + 8 * stage, nb & 1);
      const uint32_t b = b_base + stage * B_STAGE_BYTES;
      wgmma_fence();
      if (part == 0) {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) Wgmma<N, !SPLIT>::mma(d, gmma_desc(a_hi + 32 * ks), gmma_desc(b + 32 * ks), (kc | ks) != 0);
        if (SPLIT) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) Wgmma<N, !SPLIT>::mma(d, gmma_desc(a_lo + 32 * ks), gmma_desc(b + 32 * ks), 1);
        }
      } else {
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) Wgmma<N, !SPLIT>::mma(d, gmma_desc(a_hi + 32 * ks), gmma_desc(b + 32 * ks), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      mbar_arrive(bar_empty_b + 8 * stage);
      ++bi;
    }
  }
  fence_operand(d);
}

// MODE 0: every part takes the general path; 1: every part takes the lean full-width path; 2: as 1, plus the forecast's narrow
// output layer (layer_out_narrow) as the chain's last layer.
template <bool SPLIT, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1) gw_chain_tc3_kernel(const __grid_constant__ TcChain ch) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = ch.rows_per_sample, batch = ch.batch;
  const int tiles_per_sample = (rows + TILE_M - 1) / TILE_M;
  const int num_tiles = tiles_per_sample * batch;  // batch-major: tile -> (sample = tile % batch, row block = tile / batch)
  constexpr int parts = SPLIT ? 2 : 1;

  const uint32_t bar_full_b = sbase + OFF_BAR;             // [B_STAGES] bulk copy -> consumers
  const uint32_t bar_empty_b = bar_full_b + 8 * B_STAGES;  // [B_STAGES] consumers (every thread arrives) -> producer

  if (threadIdx.x == 0) {
    if (sbase & 1023u) {  // SWIZZLE_128B operand tiles must be 1 KB aligned
      if (ch.status) atomicOr(ch.status, 4);
      __trap();
    }
    for (int i = 0; i < B_STAGES; ++i) mbar_init(bar_full_b + 8 * i, 1), mbar_init(bar_empty_b + 8 * i, NUM_WORKERS);
    fence_barrier_init();
  }
  {  // per-layer column parameters -> shared memory (zero beyond n_valid)
    float* par = reinterpret_cast<float*>(smem + OFF_PAR);
    float* lnp = reinterpret_cast<float*>(smem + OFF_LNP);
    int ln_slot = 0;
    for (int l = 0; l < ch.n_layers; ++l) {
      const TcLayer& L = ch.layer[l];
      for (int c = threadIdx.x; c < 256; c += NUM_THREADS) par[l * 256 + c] = (L.bias && c < L.n_valid) ? __ldg(L.bias + c) : 0.f;
      if (L.ln_g) {
        for (int c = threadIdx.x; c < 256; c += NUM_THREADS) {
          lnp[(ln_slot * 2 + 0) * 256 + c] = (c < L.n_valid) ? __ldg(L.ln_g + c) : 0.f;
          lnp[(ln_slot * 2 + 1) * 256 + c] = (c < L.n_valid) ? __ldg(L.ln_b + c) : 0.f;
        }
        ++ln_slot;
      }
    }
  }
  if (threadIdx.x == 32) {
    // Operand range ladder (one thread; every CTA derives the same numbers from the same inputs).  m = bound of the operand
    // about to be split, s = its power-of-two scale; layer l multiplies its accumulator by wscale_inv / s and scales its own
    // result by the next s before splitting it.
    float* scl = reinterpret_cast<float*>(smem + OFF_SCL);
    float m = fmaxf(srcbound(ch.a0[0]), srcbound(ch.a0[1]));
    if (ch.a0[0].kind == SRC_GATHER_BCAST_RELU) m += ldbound(ch.a0[0].bound2);
    float sc = fit_scale(m);
    bool bad = !(m < 3.0e38f);
    scl[2 * PAR_LAYERS] = sc;
    for (int l = 0; l < ch.n_layers; ++l) {
      const TcLayer& L = ch.layer[l];
      // (an image scaled on the device carries its max|W|: its scale and gain follow from it)
      const float wa = ldbound(L.wamax);
      const float winv = L.wamax ? 1.f / tc_weight_scale(wa, ch.split ? 2 : 1) : L.wscale_inv, gain = L.wamax ? (float)L.K * wa : L.gain;
      scl[2 * l] = winv / sc;  // (a reuse_a layer multiplies the same operand: m and sc are unchanged)
      // (a LayerNorm'd row is bounded by its parameters alone, but the value it normalises must be finite too: a NaN bias there
      // would make the whole row NaN)
      const float pre = fmaf(m, gain, L.off) + srcbound(L.add[0]) + srcbound(L.add[1]);
      float mo = L.ln_g ? L.ln_bound : pre;
      mo += srcbound(L.residual);
      bad = bad || !(mo < 3.0e38f) || !(pre < 3.0e38f);
      if (blockIdx.x == 0) {
        if (L.out_bound) {  // (two layers may fill halves of one tensor: its bound is the larger one)
          const bool again = l > 0 && ch.layer[l - 1].out_bound == L.out_bound;
          *L.out_bound = again ? fmaxf(*L.out_bound, mo) : mo;
        }
        if (L.seg_bound) *L.seg_bound = mo * L.seg_maxdeg + ldbound(L.seg_add_bound);
      }
      float so = 1.f;
      if (L.feeds_next) {
        m = mo;
        sc = so = fit_scale(m);
      }
      scl[2 * l + 1] = so;
    }
    if (bad && ch.status) atomicOr(ch.status, 8);  // a magnitude bound overflowed fp32: inputs are not finite numbers of usable size
  }
  __syncthreads();
  // Register reallocation (inside each role's branch, so that ptxas budgets the roles separately)
  if (warp >= CONSUMER_WARPS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(AUX_REGS));
    if (warp == WARP_PRODUCER && lane == 0) {
      // ===================================== weight producer =========================================================
      uint32_t bi = 0;
      Tracer tr;
      tr.init(ch.trace, 0, true);
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        for (int l = 0; l < ch.n_layers; ++l) {
          const TcLayer& L = ch.layer[l];
          const uint32_t panel = (uint32_t)L.N * 128u;
          const uint8_t* w = static_cast<const uint8_t*>(L.Wp);
          const int nk = L.K >> 6;
          for (int kc = 0; kc < nk; ++kc) {
            for (int part = 0; part < parts; ++part, ++bi) {
              const uint32_t stage = bi % B_STAGES, n = bi / B_STAGES;
              mbar_wait(bar_empty_b + 8 * stage, (n & 1) ^ 1, ch.status);
              tr.ev(50 + 10 * l + 2 * kc + part);
              if (ABL3(ABL_WEIGHTS)) {
                mbar_arrive(bar_full_b + 8 * stage);
                continue;
              }
              mbar_expect_tx(bar_full_b + 8 * stage, panel);
              bulk_g2s(sbase + OFF_B + stage * B_STAGE_BYTES, w + (size_t)(kc * parts + part) * panel, panel, bar_full_b + 8 * stage);
            }
          }
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(WORKER_REGS));
  // ===================================== consumers ===================================================================
  // Warp q of warpgroup wg covers the 16 tile rows frow .. frow + 15.  A thread holds TWO CONSECUTIVE logical rows fr0, fr0 + 1
  // (operand / accumulator rows frow + lane/4 and + 8) times, in every 32-column step u, EIGHT CONSECUTIVE features
  // 32 u + fcofs .. + 7.  The 8 rows of a warp instruction are operand rows frow + 0..7 (+8): their low three bits differ, so
  // the swizzled operand stores are conflict-free.
  const int wg = warp >> 2, q = warp & 3;
  const int lr = lane >> 2, lc = lane & 3;
  const int frow = 64 * wg + 16 * q;
  const int fr0 = frow + 2 * lr;
  const int fcofs = 8 * lc;
  const uint32_t a_rows = sbase + OFF_A + 64 * wg * 128;                         // my warpgroup's operand rows
  const uint32_t fsa = sbase + OFF_A + (frow + lr) * 128 + 4 * lc + (lr << 4);  // store_operand_x4 of step 0 (step u: ^ (u & 1) << 6)
  const uint32_t wbar = 1 + wg;
  const float* scl = reinterpret_cast<const float*>(smem + OFF_SCL);
  const float a0scale = scl[2 * PAR_LAYERS];
  uint32_t bi = 0;
  float amax = 0.f;
  Tracer tr;
  tr.init(ch.trace, 5 + wg, q == 0 && lane == 0);

  auto wg_sync = [&]() GW_INLINE { asm volatile("bar.sync %0, 128;" ::"r"(wbar) : "memory"); };
  // operand rows written by my warpgroup -> visible to its wgmma (async proxy)
  auto publish = [&]() GW_INLINE {
    if (!ABL3(ABL_FENCE)) fence_proxy_async();
    wg_sync();
  };
  auto op_addr = [&](int u) GW_INLINE { return (fsa ^ ((uint32_t)(u & 1) << 6)) + (uint32_t)((u >> 1) % A_SLOTS) * A_SLOT_BYTES; };
  // ---- stage 0, general path: steps [8 w, 8 w + 8) of the operand (window w of four 64-column slots) ----------------------
  auto stage0 = [&](int tile, int w) GW_INLINE {
    const int bs = tile % batch, i0 = (tile / batch) * TILE_M;
    const int nvalid = min(TILE_M, rows - i0);
    const int r2[2] = {min(fr0, nvalid - 1), min(fr0 + 1, nvalid - 1)};
    const int nu = min(2 * (ch.K0 >> 6), 8 * w + 8), w0 = ch.a0[0].width;
    for (int u = 8 * w; u < nu; ++u) {
      const int colc = 32 * u;
      const int which = colc < w0 ? 0 : 1;
      const RowSrc& src = ch.a0[which];
      const int rel = which ? colc - w0 : colc;
      float cur[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) cur[i] = 0.f;
      if (src.kind != SRC_NONE && rel < src.width && !ABL3(ABL_LOADS)) {
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          load8(src_row(src, bs, i0, r2[m]), rel + fcofs, src.width, cur + 8 * m);
          if (src.kind == SRC_GATHER_BCAST_RELU) {
            float t[8];
            load8(src.base2 + (size_t)(uint32_t)(i0 + r2[m]) * (size_t)src.ld2, rel + fcofs, src.width, t);
#pragma unroll
            for (int k = 0; k < 8; ++k) cur[8 * m + k] = fmaxf(cur[8 * m + k] + t[k], 0.f);
          }
        }
      }
      if (a0scale != 1.f) {
#pragma unroll
        for (int i = 0; i < 16; ++i) cur[i] *= a0scale;
      }
      if (!ABL3(ABL_CONVERT)) store_operand_x4<SPLIT, true>(op_addr(u), cur, amax);
    }
    publish();
  };

  // ---- stage 0, lean path: NC0 + NC1 64-column chunks from one or two aligned sources, window W (chunks 4 W .. 4 W + 3) ------
  // The rows stream from HBM (edge state) or L2 (node state): up to four steps (16 x LDG.128 per thread) are in flight before the
  // first one is converted.  GBR: the operand is relu(gathered row + broadcast row); the two tables are kept apart until the step
  // is converted (two steps in flight).
  auto stage0_fast = [&](auto NC0c, auto NC1c, auto GBRc, auto Wc, int tile) GW_INLINE {
    constexpr int NC0 = decltype(NC0c)::value, NC1 = decltype(NC1c)::value, NC = NC0 + NC1;
    constexpr bool GBR = decltype(GBRc)::value != 0;
    constexpr int U0 = 8 * decltype(Wc)::value, U1 = (2 * NC < U0 + 8) ? 2 * NC : U0 + 8;
    constexpr int DEPTH = GBR ? 2 : 4;
    const int bs = tile % batch, i0 = (tile / batch) * TILE_M;
    const int nvalid = min(TILE_M, rows - i0);
    const int r2[2] = {min(fr0, nvalid - 1), min(fr0 + 1, nvalid - 1)};
    const char* pa[2];
    const char* pb[2] = {nullptr, nullptr};  // second source, or the broadcast table of GBR
    row_ptrs2(ch.a0[0], bs, i0, r2, fcofs, pa);
    if constexpr (GBR) {
#pragma unroll
      for (int m = 0; m < 2; ++m) pb[m] = reinterpret_cast<const char*>(ch.a0[0].base2 + (size_t)(uint32_t)(i0 + r2[m]) * (size_t)ch.a0[0].ld2 + fcofs);
    } else if constexpr (NC1 > 0) {
      row_ptrs2(ch.a0[1], bs, i0, r2, fcofs, pb);
    }
    float buf[DEPTH][16] = {};  // [row m][8 features]
    float bufb[GBR ? DEPTH : 1][16] = {};
    auto fetch = [&](auto uu) GW_INLINE {
      constexpr int u = decltype(uu)::value, k = (u - U0) % DEPTH;
      if (ABL3(ABL_LOADS)) return;
      if constexpr (GBR) {
        ld256(pa[0] + 128 * u, buf[k]), ld256(pa[1] + 128 * u, buf[k] + 8);
        ld256(pb[0] + 128 * u, bufb[k]), ld256(pb[1] + 128 * u, bufb[k] + 8);
      } else if constexpr (u < 2 * NC0) {
        ld256(pa[0] + 128 * u, buf[k]), ld256(pa[1] + 128 * u, buf[k] + 8);
      } else {
        ld256(pb[0] + 128 * (u - 2 * NC0), buf[k]), ld256(pb[1] + 128 * (u - 2 * NC0), buf[k] + 8);
      }
    };
    static_for<U0, (U1 < U0 + DEPTH ? U1 : U0 + DEPTH)>([&](auto uu) GW_INLINE { fetch(uu); });
    static_for<U0, U1>([&](auto uu) GW_INLINE {
      constexpr int u = decltype(uu)::value, k = (u - U0) % DEPTH;
      float(&cur)[16] = buf[k];
      if constexpr (GBR) {
#pragma unroll
        for (int i = 0; i < 16; ++i) cur[i] = fmaxf(cur[i] + bufb[k][i], 0.f);
      }
      if (a0scale != 1.f) {
#pragma unroll
        for (int i = 0; i < 16; ++i) cur[i] *= a0scale;
      }
      if (!ABL3(ABL_CONVERT)) store_operand_x4<SPLIT, true>(op_addr(u), cur, amax);
      if constexpr (u + DEPTH < U1) fetch(ic<u + DEPTH>{});  // refill the buffer just consumed
    });
    publish();
  };

  // scale + bias of the accumulator in place, steps [0, nu)
  auto bias_in_place = [&](float (&acc)[128], int l, int nu, float wsi) GW_INLINE {
    const uint32_t bias_a = sbase + OFF_PAR + l * 1024 + 4 * fcofs;
    static_for<0, 8>([&](auto uu) GW_INLINE {
      constexpr int u = decltype(uu)::value;
      if (u < nu) {
        const float4 bl = lds128(bias_a + 128 * u), bh = lds128(bias_a + 128 * u + 16);
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[16 * u + i] = fmaf(acc[16 * u + i], wsi, col8(bl, bh, i));
      }
    });
  };
  // LayerNorm statistics of my two rows over their nval real columns (two passes over the registers; the four lanes of a row
  // combine with two shuffles): v -> v * rs[m] + sh[m]
  auto ln_stats = [&](float (&acc)[128], int nu, int nval, float (&rs)[2], float (&sh)[2]) GW_INLINE {
    float s[2] = {0.f, 0.f};
    static_for<0, 8>([&](auto uu) GW_INLINE {
      constexpr int u = decltype(uu)::value;
      if (u < nu) {
#pragma unroll
        for (int i = 0; i < 16; ++i) s[(i >> 1) & 1] += acc[16 * u + i];  // (columns beyond nval are exactly zero)
      }
    });
#pragma unroll
    for (int m = 0; m < 2; ++m) s[m] += __shfl_xor_sync(0xffffffffu, s[m], 1), s[m] += __shfl_xor_sync(0xffffffffu, s[m], 2);
    const float inv = 1.0f / (float)nval;
    const float mean[2] = {s[0] * inv, s[1] * inv};
    float v2[2] = {0.f, 0.f};
    static_for<0, 8>([&](auto uu) GW_INLINE {
      constexpr int u = decltype(uu)::value;
      if (u < nu) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int m = (i >> 1) & 1;
          const float d = (32 * u + fcofs + 2 * (i >> 2) + (i & 1) < nval) ? acc[16 * u + i] - mean[m] : 0.f;
          v2[m] = fmaf(d, d, v2[m]);
        }
      }
    });
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      v2[m] += __shfl_xor_sync(0xffffffffu, v2[m], 1), v2[m] += __shfl_xor_sync(0xffffffffu, v2[m], 2);
      const float rstd = 1.0f / sqrtf(v2[m] * inv + 1e-5f);
      rs[m] = rstd, sh[m] = -mean[m] * rstd;
    }
  };

  // ---- one layer's epilogue, lean path: N = 64 NP, full-width aligned addends / residual / output ---------------------------
  // Accumulator fragments are in fragment order (index 4 g + 2 m + e = row m, feature 2 g + e), everything read from / written
  // to global memory in row order (index 8 m + t); FR() / PX() translate at compile time.  The global operands of step u + 1 are
  // in flight while step u is stored / converted.
  auto layer_fast = [&](float (&acc)[128], auto FLc, auto NPc, int l, int tile, int ln_slot) GW_INLINE {
    constexpr int F = decltype(FLc)::value, NP = decltype(NPc)::value, NU = 2 * NP;
    constexpr bool has_add0 = (F & F_ADD0) != 0, has_add1 = (F & F_ADD1) != 0, has_res = (F & F_RES) != 0, has_out = (F & F_OUT) != 0;
    constexpr bool relu = (F & F_RELU) != 0, has_ln = (F & F_LN) != 0, feeds = (F & F_FEEDS) != 0, has_seg = (F & F_SEG) != 0;
    constexpr bool has0 = has_add0 || has_res;
    const TcLayer& L = ch.layer[l];
    const int bs = tile % batch, i0 = (tile / batch) * TILE_M;
    const int nvalid = min(TILE_M, rows - i0);
    const float wsi = scl[2 * l], osc = scl[2 * l + 1];
    const uint32_t g_a = sbase + OFF_LNP + 4 * fcofs + (ln_slot * 2) * 1024, b_a = g_a + 1024;
    const RowSrc& src0 = has_add0 ? L.add[0] : L.residual;
    const char* p0[2] = {nullptr, nullptr};  // addend 0 or residual rows
    const char* p1[2] = {nullptr, nullptr};  // addend 1 rows
    float pf0[16] = {}, pf1[16] = {};
    const bool ld_on = !ABL3(ABL_LOADS);
    auto ld2 = [&](const char* const(&p)[2], int off, float(&o)[16]) GW_INLINE { ld256(p[0] + off, o), ld256(p[1] + off, o + 8); };
    {
      const int r2[2] = {min(fr0, nvalid - 1), min(fr0 + 1, nvalid - 1)};
      if constexpr (has0) row_ptrs2(src0, bs, i0, r2, fcofs, p0);
      if constexpr (has_add1) row_ptrs2(L.add[1], bs, i0, r2, fcofs, p1);
    }
    if constexpr (has0) {
      if (ld_on) ld2(p0, 0, pf0);
    }
    if constexpr (has_add1) {
      if (ld_on) ld2(p1, 0, pf1);
    }
    // targets of my rows (fused per-target sums)
    int d0 = 0, d1 = 0, dprev_g = 0;
    if constexpr (has_seg) {
      const int32_t* sd = L.seg_dst + i0;
      d0 = (fr0 < nvalid) ? __ldg(sd + fr0) : -1;
      d1 = (fr0 + 1 < nvalid) ? __ldg(sd + fr0 + 1) : -2;
      dprev_g = (lr == 0 && i0 + frow > 0 && frow < nvalid) ? __ldg(sd + frow - 1) : -8;
    }
    bias_in_place(acc, l, NU, wsi);
    float rs[2] = {1.f, 1.f}, sh[2] = {0.f, 0.f};  // LayerNorm as v * rs[m] + sh[m] per row
    if constexpr (has_ln) {
      if (!ABL3(ABL_LN)) ln_stats(acc, NU, 64 * NP, rs, sh);
    }
    // output rows (fp32): my two rows are ldo apart
    char* po = nullptr;
    const size_t ostr = 4 * (size_t)L.ldo;
    const bool st0 = fr0 < nvalid, st1 = fr0 + 1 < nvalid;
    if constexpr (has_out) po = reinterpret_cast<char*>(L.out + ((size_t)bs * rows + i0 + fr0) * (size_t)L.ldo + fcofs);
    // Fused per-target sums.  Rows are sorted by target, a target's rows are a run of at most 8 consecutive rows.  The 8 lane
    // groups of a warp hold 16 consecutive rows, two per thread.  The thread in which a run STARTS owns it: it adds to its own
    // rows of the run the heads H (the rows before the first boundary) of the following threads the run reaches into, and
    // stores the sum.  The heads are chained by doubling: G1(t) = H(t) + k(t) H(t+1) where k(t) = "the run passes through
    // thread t into t+1"; the owner takes H(t+1) and G1(t+2) (two shuffles per value reach four threads = 7 rows; a third,
    // G2(t+4), reaches the fifth thread an 8-row run can touch).  A run that reaches the next 16-row group continues there; that
    // group's first thread leaves the continuation in the carry buffer (gw_seg_carry_kernel adds it to the run's row afterwards).
    bool bb = false, tail_st = false, head_st = false, one_st = false, one_any = false, deep = false;
    float mbf = 1.f, c1f = 0.f, e2f = 0.f, e4f = 0.f, kf = 0.f, k1f = 0.f;
    char* tail_p = nullptr;
    char* carry_p = nullptr;
    const char* add_p = nullptr;
    if constexpr (has_seg) {
      int dprev = __shfl_up_sync(0xffffffffu, d1, 4);
      if (lr == 0) dprev = dprev_g;
      const bool ba = d0 != dprev;  // my first row starts a run
      bb = d1 != d0;                // my second row starts a run
      mbf = bb ? 0.f : 1.f;
      const uint32_t nba = __shfl_down_sync(0xffffffffu, (uint32_t)ba, 4);
      const bool c1 = lr < 7 && !nba;  // my last run continues into the next thread's rows
      const bool k = c1 && !bb;        // ... and it entered my rows from the left or at my first row: it passes THROUGH me
      const uint32_t k1 = __shfl_down_sync(0xffffffffu, (uint32_t)k, 4), k2 = __shfl_down_sync(0xffffffffu, (uint32_t)k, 8);
      const uint32_t k3 = __shfl_down_sync(0xffffffffu, (uint32_t)k, 12);
      const bool e2 = c1 && k1;         // (k(t+1) implies lane group t+2 exists)
      const bool e4 = e2 && k2 && k3;
      c1f = c1 ? 1.f : 0.f, e2f = e2 ? 1.f : 0.f, e4f = e4 ? 1.f : 0.f, kf = k ? 1.f : 0.f, k1f = (k && k1) ? 1.f : 0.f;
      deep = L.seg_maxdeg > 7;  // (a run of 8 rows can reach the fifth thread; 7 rows end in the fourth)
      carry_p = reinterpret_cast<char*>(L.seg_carry + ((((size_t)bs * tiles_per_sample + (size_t)(i0 / TILE_M)) * 8 + (size_t)(frow >> 4)) * 256 + fcofs));
      // the run that ends with (or passes through) my second row: mine to store if it starts in my rows; the group's first
      // thread stores the continuation of the previous group's run into the carry buffer
      if (ba || bb) {
        tail_st = d1 >= 0;
        tail_p = reinterpret_cast<char*>(L.seg_out + ((size_t)bs * L.seg_rows + (size_t)(uint32_t)max(d1, 0)) * (size_t)L.seg_ld + fcofs);
      } else if (lr == 0) {
        tail_st = d1 >= 0;
        tail_p = carry_p;
      }
      head_st = lr == 0 && !ba && bb && d0 >= 0;  // the previous group's run ends with my first row
      one_st = ba && bb && d0 >= 0;               // my first row is a run of its own (a target with a single row)
      one_any = __any_sync(0xffffffffu, one_st);
      // per-target constant (a constant residual summed over the target's rows, once per weight set): the owner of a run adds it
      if (L.seg_add && (ba || bb) && d1 >= 0)
        add_p = reinterpret_cast<const char*>(L.seg_add + (size_t)(uint32_t)d1 * (size_t)L.seg_ld + fcofs);
    }
    static_for<0, NU>([&](auto uu) GW_INLINE {
      constexpr int u = decltype(uu)::value;
      float v[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = acc[16 * u + i];
      [[maybe_unused]] float sadd[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if constexpr (has_seg) {
        if (add_p) ld256(add_p + 128 * u, sadd);
      }
      if constexpr (has_add0) {
        if (ld_on) {
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] += pf0[PX(i)];
        }
      }
      if constexpr (has_add1) {
        if (ld_on) {
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] += pf1[PX(i)];
        }
      }
      if constexpr (relu) {
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i], 0.f);
      }
      if constexpr (has_ln) {
        const float4 gl = lds128(g_a + 128 * u), gh = lds128(g_a + 128 * u + 16);
        const float4 el = lds128(b_a + 128 * u), eh = lds128(b_a + 128 * u + 16);
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int m = (i >> 1) & 1;
          v[i] = fmaf(fmaf(v[i], rs[m], sh[m]), col8(gl, gh, i), col8(el, eh, i));
        }
      }
      if constexpr (has_res) {
        if (ld_on) {
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] += pf0[PX(i)];
        }
      }
      if constexpr (u + 1 < NU) {  // next step's global operands: in flight while this step is stored / converted
        if constexpr (has0) {
          if (ld_on) ld2(p0, 128 * (u + 1), pf0);
        }
        if constexpr (has_add1) {
          if (ld_on) ld2(p1, 128 * (u + 1), pf1);
        }
      }
      if constexpr (has_out) {
        if (!ABL3(ABL_STORES)) {
          if (st0) st256(po + 128 * u, v[FR(0, 0)], v[FR(0, 1)], v[FR(0, 2)], v[FR(0, 3)], v[FR(0, 4)], v[FR(0, 5)], v[FR(0, 6)], v[FR(0, 7)]);
          if (st1) st256(po + ostr + 128 * u, v[FR(1, 0)], v[FR(1, 1)], v[FR(1, 2)], v[FR(1, 3)], v[FR(1, 4)], v[FR(1, 5)], v[FR(1, 6)], v[FR(1, 7)]);
        }
      }
      if constexpr (has_seg) {
        float T[8], H[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float xa = v[FR(0, t)], xb = v[FR(1, t)];
          T[t] = fmaf(mbf, xa, xb);  // the run through my second row: both rows, or the second alone after a boundary
          H[t] = bb ? xa : T[t];     // my rows before the first boundary: what the owner of the run that reaches me adds
        }
        const bool sts_on = !ABL3(ABL_STORES);
        if (head_st && sts_on) st256(carry_p + 128 * u, H[0], H[1], H[2], H[3], H[4], H[5], H[6], H[7]);
        if (one_any) {
          if (one_st && sts_on) {
            char* dp = reinterpret_cast<char*>(L.seg_out + ((size_t)bs * L.seg_rows + (size_t)(uint32_t)d0) * (size_t)L.seg_ld + fcofs);
            float a1[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (L.seg_add) ld256(reinterpret_cast<const char*>(L.seg_add + (size_t)(uint32_t)d0 * (size_t)L.seg_ld + fcofs) + 128 * u, a1);
            st256(dp + 128 * u, H[0] + a1[0], H[1] + a1[1], H[2] + a1[2], H[3] + a1[3], H[4] + a1[4], H[5] + a1[5], H[6] + a1[6], H[7] + a1[7]);
          }
        }
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float h1 = __shfl_down_sync(0xffffffffu, H[t], 4);
          T[t] = fmaf(c1f, h1, T[t]);
          H[t] = fmaf(kf, h1, H[t]);  // G1
        }
#pragma unroll
        for (int t = 0; t < 8; ++t) T[t] = fmaf(e2f, __shfl_down_sync(0xffffffffu, H[t], 8), T[t]);
        if (deep) {
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            const float g2 = fmaf(k1f, __shfl_down_sync(0xffffffffu, H[t], 8), H[t]);  // G2
            T[t] = fmaf(e4f, __shfl_down_sync(0xffffffffu, g2, 16), T[t]);
          }
        }
        if (tail_st && sts_on)  // (sadd is zero for the threads that write a carry row or own no run)
          st256(tail_p + 128 * u, T[0] + sadd[0], T[1] + sadd[1], T[2] + sadd[2], T[3] + sadd[3], T[4] + sadd[4], T[5] + sadd[5], T[6] + sadd[6],
                T[7] + sadd[7]);
      }
      if constexpr (feeds) {
        if (osc != 1.f) {
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] *= osc;
        }
        if (!ABL3(ABL_CONVERT)) store_operand_x4<SPLIT, false>(op_addr(u), v, amax);
      }
      tr.ev(700 + 10 * l + u);
    });
    if constexpr (feeds) publish();
  };

  // ---- the forecast's output layer on the lean path ---------------------------------------------------------------------------
  // N is padded to 64 k columns of which n_valid (78) are real; the rows of the output and of the residual (the start features)
  // are only 8-byte aligned: 64-bit accesses, one pair of columns at a time, steps beyond n_valid idle.  Keeping this layer in the
  // node chain saves the hidden rows' round trip through HBM and a general-path chain per step.
  auto layer_out_narrow = [&](float (&acc)[128], int l, int tile) GW_INLINE {
    const TcLayer& L = ch.layer[l];
    const int bs = tile % batch, i0 = (tile / batch) * TILE_M;
    const int nvalid = min(TILE_M, rows - i0);
    const int nu = L.N >> 5, nval = L.n_valid;
    const bool has_res = L.residual.kind != SRC_NONE;
    const float* rp[2] = {nullptr, nullptr};
    if (has_res) {
      const float* base = reinterpret_cast<const float*>(src_sample_base(L.residual, bs));
#pragma unroll
      for (int m = 0; m < 2; ++m) rp[m] = base + (size_t)(uint32_t)(i0 + min(fr0 + m, nvalid - 1)) * (size_t)L.residual.ld;
    }
    float* op[2];
#pragma unroll
    for (int m = 0; m < 2; ++m) op[m] = L.out + ((size_t)bs * rows + i0 + fr0 + m) * (size_t)L.ldo;
    const bool st[2] = {fr0 < nvalid, fr0 + 1 < nvalid};
    bias_in_place(acc, l, nu, scl[2 * l]);
    static_for<0, 8>([&](auto uu) GW_INLINE {
      constexpr int u = decltype(uu)::value;
      const int c0 = 32 * u + fcofs;
      if (u < nu && 32 * u < nval) {  // warp-uniform: this step holds real features
        float2 r[2][4] = {};
        if (has_res && !ABL3(ABL_LOADS)) {
#pragma unroll
          for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int g = 0; g < 4; ++g)
              if (c0 + 2 * g < nval) r[m][g] = __ldg(reinterpret_cast<const float2*>(rp[m] + c0 + 2 * g));
        }
        if (!ABL3(ABL_STORES)) {
#pragma unroll
          for (int m = 0; m < 2; ++m)
#pragma unroll
            for (int g = 0; g < 4; ++g)
              if (st[m] && c0 + 2 * g < nval)  // (n_valid is even: a pair is inside or outside as a whole)
                *reinterpret_cast<float2*>(op[m] + c0 + 2 * g) =
                    make_float2(acc[16 * u + 4 * g + 2 * m] + r[m][g].x, acc[16 * u + 4 * g + 2 * m + 1] + r[m][g].y);
        }
      }
    });
  };

  // ---- one layer's epilogue, general path: any N (multiple of 64 in the perm32 image), n_valid real columns, sources and outputs
  // of any width and alignment ---------------------------------------------------------------------------------------------------
  auto layer_gen = [&](float (&acc)[128], int l, int tile, int ln_slot, bool last_layer) GW_INLINE {
    const TcLayer& L = ch.layer[l];
    const int bs = tile % batch, i0 = (tile / batch) * TILE_M;
    const int nvalid = min(TILE_M, rows - i0);
    const int nu = L.N >> 5, nval = L.n_valid;
    const float osc = scl[2 * l + 1];
    const bool has_add0 = L.add[0].kind != SRC_NONE, has_add1 = L.add[1].kind != SRC_NONE;
    const bool has_res = L.residual.kind != SRC_NONE, has_out = L.out != nullptr;
    const bool relu = L.relu != 0, feeds = L.feeds_next != 0, has_ln = L.ln_g != nullptr;
    const bool has_mask = L.mask.kind != SRC_NONE, has_pre = L.save_pre != nullptr;
    const uint32_t g_a = sbase + OFF_LNP + 4 * fcofs + (ln_slot * 2) * 1024, b_a = g_a + 1024;
    const int r2[2] = {min(fr0, nvalid - 1), min(fr0 + 1, nvalid - 1)};
    const float* q0[2] = {nullptr, nullptr};  // addend 0 / residual rows
    const float* q1[2] = {nullptr, nullptr};  // addend 1 rows
    const RowSrc& src0 = has_add0 ? L.add[0] : L.residual;
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      if (has_add0 || has_res) q0[m] = src_row(src0, bs, i0, r2[m]);
      if (has_add1) q1[m] = src_row(L.add[1], bs, i0, r2[m]);
    }
    // plain fp32 stores of my two rows' 8 features (out / save_pre): 128-bit where the row allows it
    auto store8 = [&](float* base, const float (&v)[16], int col) GW_INLINE {
#pragma unroll
      for (int m = 0; m < 2; ++m) {
        if (fr0 + m < nvalid) {
          float* orow = base + ((size_t)bs * rows + i0 + fr0 + m) * (size_t)L.ldo + col;
          if (col + 8 <= L.out_cols && (reinterpret_cast<uintptr_t>(orow) & 15) == 0) {
            *reinterpret_cast<float4*>(orow) = make_float4(v[FR(m, 0)], v[FR(m, 1)], v[FR(m, 2)], v[FR(m, 3)]);
            *reinterpret_cast<float4*>(orow + 4) = make_float4(v[FR(m, 4)], v[FR(m, 5)], v[FR(m, 6)], v[FR(m, 7)]);
          } else {
#pragma unroll
            for (int k = 0; k < 8; ++k)
              if (col + k < L.out_cols) orow[k] = v[FR(m, k)];
          }
        }
      }
    };
    bias_in_place(acc, l, nu, scl[2 * l]);
    float rs[2] = {1.f, 1.f}, sh[2] = {0.f, 0.f};
    if (has_ln && !ABL3(ABL_LN)) ln_stats(acc, nu, nval, rs, sh);
    // where the values go: this GPU's memory, or (last layer of the forecast chain on a multi-GPU job) every GPU's gather buffer at
    // once -- NVLink multicast or one store per peer mapping
    const int omode = last_layer ? ch.out_mode : 0;
    const ptrdiff_t mc_delta = reinterpret_cast<const char*>(ch.out_mc) - reinterpret_cast<const char*>(L.out);
    auto put4 = [&](float* p, float a, float b, float c, float d) GW_INLINE {
      if (omode == 0) {
        *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
      } else if (omode == 1) {
        asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(reinterpret_cast<char*>(p) + mc_delta), "f"(a), "f"(b),
                     "f"(c), "f"(d)
                     : "memory");
      } else {
        for (int j = 0; j < ch.n_out_peers; ++j)
          *reinterpret_cast<float4*>(reinterpret_cast<char*>(p) + (reinterpret_cast<const char*>(ch.out_peer[j]) - reinterpret_cast<const char*>(L.out))) =
              make_float4(a, b, c, d);
      }
    };
    auto put1 = [&](float* p, float a) GW_INLINE {
      if (omode == 0) {
        *p = a;
      } else if (omode == 1) {
        asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(reinterpret_cast<char*>(p) + mc_delta), "f"(a) : "memory");
      } else {
        for (int j = 0; j < ch.n_out_peers; ++j)
          *reinterpret_cast<float*>(reinterpret_cast<char*>(p) + (reinterpret_cast<const char*>(ch.out_peer[j]) - reinterpret_cast<const char*>(L.out))) = a;
      }
    };
    static_for<0, 8>([&](auto uu) GW_INLINE {
      constexpr int u = decltype(uu)::value;
      if (u < nu) {
        const int col = 32 * u + fcofs;
        const bool ld_ok = !ABL3(ABL_LOADS);
        float v[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = acc[16 * u + i];
        float t[16];
        if (has_add0 && ld_ok) {
          load8(q0[0], col, src0.width, t), load8(q0[1], col, src0.width, t + 8);
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] += t[PX(i)];
        }
        if (has_add1 && ld_ok) {
          load8(q1[0], col, L.add[1].width, t), load8(q1[1], col, L.add[1].width, t + 8);
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] += t[PX(i)];
        }
        if (relu) {
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] = fmaxf(v[i], 0.f);
        }
        if (has_pre && !ABL3(ABL_STORES)) store8(L.save_pre, v, col);  // the value entering LayerNorm
        if (has_ln) {
          const float4 gl = lds128(g_a + 128 * u), gh = lds128(g_a + 128 * u + 16);
          const float4 el = lds128(b_a + 128 * u), eh = lds128(b_a + 128 * u + 16);
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int m = (i >> 1) & 1;
            v[i] = fmaf(fmaf(v[i], rs[m], sh[m]), col8(gl, gh, i), col8(el, eh, i));
          }
        }
        if (!has_add0 && has_res && ld_ok) {
          load8(q0[0], col, src0.width, t), load8(q0[1], col, src0.width, t + 8);
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] += t[PX(i)];
        }
        if (has_mask) {  // the ReLU's backward: keep where the mask row (the taped activation) is positive
          load8(src_row(L.mask, bs, i0, r2[0]), col, L.mask.width, t), load8(src_row(L.mask, bs, i0, r2[1]), col, L.mask.width, t + 8);
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] = t[PX(i)] > 0.f ? v[i] : 0.f;
        }
        if (nval < L.N) {  // padded output columns (e.g. 78 of 128) must stay exactly zero
#pragma unroll
          for (int i = 0; i < 16; ++i)
            if (col + 2 * (i >> 2) + (i & 1) >= nval) v[i] = 0.f;
        }
        if (has_out && !ABL3(ABL_STORES)) {
#pragma unroll
          for (int m = 0; m < 2; ++m) {
            if (fr0 + m < nvalid) {
              float* orow = L.out + ((size_t)bs * rows + i0 + fr0 + m) * (size_t)L.ldo + col;
              if (col + 8 <= L.out_cols && (reinterpret_cast<uintptr_t>(orow) & 15) == 0) {
                put4(orow, v[FR(m, 0)], v[FR(m, 1)], v[FR(m, 2)], v[FR(m, 3)]);
                put4(orow + 4, v[FR(m, 4)], v[FR(m, 5)], v[FR(m, 6)], v[FR(m, 7)]);
              } else {
#pragma unroll
                for (int k = 0; k < 8; ++k)
                  if (col + k < L.out_cols) put1(orow + k, v[FR(m, k)]);
              }
            }
          }
        }
        if (feeds) {
          if (osc != 1.f) {
#pragma unroll
            for (int i = 0; i < 16; ++i) v[i] *= osc;
          }
          if (!ABL3(ABL_CONVERT)) store_operand_x4<SPLIT, false>(op_addr(u), v, amax);
        }
      }
    });
    if (feeds) publish();
  };

  // One layer of the chain on the tile: its product (N, the wgmma shape, at compile time) and its epilogue.
  auto run_layer = [&](auto Nc, int l, int tile, int ln_slot) GW_INLINE {
    constexpr int N = decltype(Nc)::value;
    const TcLayer& L = ch.layer[l];
    float acc[128];  // (per layer: the first wgmma of the layer overwrites it, so nothing is live across stage 0)
    auto mma = [&](int kc0, int kc1) GW_INLINE {
      tr.ev(100 + kc0);
      mma_chunks<SPLIT, N>(acc, a_rows, sbase + OFF_B, bar_full_b, bar_empty_b, bi, kc0, kc1);
      wg_sync();  // every wgmma of my warpgroup has read its operand: the epilogue may overwrite it
      tr.ev(110 + kc0);
    };
    if (l == 0) {
      // stage 0 in windows of A_SLOTS chunks, each multiplied as soon as it is assembled
      const int nk0 = ch.K0 >> 6;
      for (int w = 0; 4 * w < nk0; ++w) {
        tr.ev(480 + w);
        if constexpr (MODE >= 1) {
          if (ch.a0[1].kind != SRC_NONE) {  // node chains: [x | aggregate]
            if (w == 0) stage0_fast(ic<4>{}, ic<4>{}, ic<0>{}, ic<0>{}, tile);
            else stage0_fast(ic<4>{}, ic<4>{}, ic<0>{}, ic<1>{}, tile);
          } else if (ch.a0[0].kind == SRC_GATHER_BCAST_RELU) {
            stage0_fast(ic<4>{}, ic<0>{}, ic<1>{}, ic<0>{}, tile);  // decoder edges
          } else if (ch.K0 == 256) {
            stage0_fast(ic<4>{}, ic<0>{}, ic<0>{}, ic<0>{}, tile);  // edge chains, products of x
          } else {
            stage0_fast(ic<2>{}, ic<0>{}, ic<0>{}, ic<0>{}, tile);  // widened feature rows (K0 = 128)
          }
        } else {
          stage0(tile, w);
        }
        mma(4 * w, min(nk0, 4 * w + 4));
      }
    } else {
      mma(0, L.K >> 6);  // the operand the previous layer left (or, reuse_a, the one it multiplied)
    }
    if constexpr (MODE >= 1) {
      if constexpr (MODE == 2) {  // (a kernel of its own: only the chain that ends in the forecast's output layer carries it)
        if (L.kind & F_NARROW) {
          layer_out_narrow(acc, l, tile);
          return;
        }
      }
#define GW_LF(M, NP_) case (M): layer_fast(acc, ic<(M)>{}, ic<(NP_)>{}, l, tile, ln_slot); break
      if constexpr (N == 256) {
        switch (L.kind) {
          GW_LF(F_ADD0 | F_ADD1 | F_RELU | F_FEEDS, 4);  // edge layer 1: gathered P[src] + P[dst]
          GW_LF(F_ADD0 | F_RELU | F_FEEDS, 4);           // encoder edge layer 1: broadcast constant term
          GW_LF(F_RELU | F_FEEDS, 4);                    // hidden layers
          GW_LF(F_LN | F_RES | F_OUT, 4);                // last layer of an edge / node MLP
          GW_LF(F_LN | F_RES | F_OUT | F_SEG, 4);        // ... of the processor's edge MLP: e' rows and their per-node sums
          GW_LF(F_LN | F_RES | F_SEG, 4);                // ... of the decoder's edge MLP: per-point sums only, e' is never written
          GW_LF(F_LN | F_SEG, 4);                        // ... with its constant residual hoisted into a per-point constant (seg_add)
          GW_LF(F_LN | F_RES | F_OUT | F_FEEDS, 4);      // ... whose rows are also the operand of the next block's P products
          GW_LF(F_LN | F_FEEDS, 4);                      // LayerNorm feeding the next MLP of the same chain
          GW_LF(F_OUT, 4);                               // per-node products P = x W^T
          GW_LF(F_RELU | F_OUT, 4);
          default: break;  // (the launcher sends chains with any other layer to the general path)
        }
      } else {
        switch (L.kind) {
          GW_LF(F_RELU | F_FEEDS, 2);  // hidden layers of the node decoder (N = 128)
          GW_LF(F_RELU | F_OUT, 2);
          default: break;
        }
      }
#undef GW_LF
    } else {
      layer_gen(acc, l, tile, ln_slot, l + 1 == ch.n_layers);
    }
  };

  const int n_layers = ch.n_layers;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int ln_slot = 0;
    for (int l = 0; l < n_layers; ++l) {
      const int N = ch.layer[l].N;  // (64 / 128 / 192 / 256; the lean path has 128 and 256 only)
      if constexpr (MODE >= 1) {
        if (N == 256) run_layer(ic<256>{}, l, tile, ln_slot);
        else run_layer(ic<128>{}, l, tile, ln_slot);
      } else {
        if (N == 256) run_layer(ic<256>{}, l, tile, ln_slot);
        else if (N == 192) run_layer(ic<192>{}, l, tile, ln_slot);
        else if (N == 128) run_layer(ic<128>{}, l, tile, ln_slot);
        else run_layer(ic<64>{}, l, tile, ln_slot);
      }
      if (ch.layer[l].ln_g) ++ln_slot;
      tr.ev(900 + l);
    }
  }
  if (SPLIT && ch.status && amax > 60000.f) atomicOr(ch.status, 1);  // operand left the fp16 range: results invalid
}

}  // namespace t3

static bool aligned32(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 31) == 0; }
static bool simple_kind(int k) { return k == SRC_STREAM || k == SRC_BCAST || k == SRC_GATHER || k == SRC_BGATHER; }
// a source every thread may read with 8-byte loads over `need` columns
// byte offsets inside a fast-path source fit 32 bits: gathered rows are addressed relative to the sample, contiguous rows
// relative to the tile
static bool fits32(const RowSrc& s) {
  const bool g = s.kind == SRC_GATHER || s.kind == SRC_BGATHER || s.kind == SRC_GATHER_BCAST_RELU;
  const long long span = g ? (long long)s.src_rows : 128;
  return span * (long long)s.ld * 4 + 4096 < (1ll << 32);
}
static bool src_fast(const RowSrc& s, int need) {
  return simple_kind(s.kind) && s.width >= need && aligned32(s.base + s.col0) && !(s.ld & 7) && fits32(s);  // 32-byte row segments
}

// Marks which parts of a chain take the lean full-width path (ch.fast) and the epilogue kind of every layer.
static void tc3_mark_lean(TcChain& ch) {
  using namespace t3;
  ch.fast = 0;
  {  // stage 0: one 128- or 256-wide aligned source, or two 256-wide ones (the shapes stage0_fast is instantiated for)
    bool ok = true;
    int wsum = 0;
    for (int a = 0; a < 2; ++a) {
      const RowSrc& s = ch.a0[a];
      if (s.kind == SRC_NONE) continue;
      const bool gbr = s.kind == SRC_GATHER_BCAST_RELU;
      ok = ok && (simple_kind(s.kind) || gbr) && aligned32(s.base + s.col0) && !(s.ld & 7);  // 32-byte row segments
      if (gbr) ok = ok && aligned32(s.base2) && !(s.ld2 & 7);
      wsum += s.width;
    }
    const bool two = ch.a0[1].kind != SRC_NONE;
    ok = ok && ch.a0[0].kind != SRC_NONE && wsum == ch.K0;
    ok = ok && (two ? (ch.a0[0].width == 256 && ch.a0[1].width == 256) : (ch.K0 == 256 || ch.K0 == 128));
    if (ch.a0[0].kind == SRC_GATHER_BCAST_RELU) ok = ok && !two && ch.K0 == 256;
    if (ok) ch.fast |= (int32_t)0x80000000u;
  }
  static const int kinds4[] = {F_ADD0 | F_ADD1 | F_RELU | F_FEEDS, F_ADD0 | F_RELU | F_FEEDS, F_RELU | F_FEEDS, F_LN | F_RES | F_OUT,
                               F_LN | F_RES | F_OUT | F_SEG, F_LN | F_RES | F_SEG, F_LN | F_SEG, F_LN | F_RES | F_OUT | F_FEEDS, F_LN | F_FEEDS, F_OUT,
                               F_RELU | F_OUT};
  static const int kinds2[] = {F_RELU | F_FEEDS, F_RELU | F_OUT};
  for (int l = 0; l < ch.n_layers; ++l) {
    const TcLayer& L = ch.layer[l];
    // the training step's epilogue parts (pre-LayerNorm store, ReLU mask) exist on the general path only: such a layer must not
    // take the narrow output layer below either, whose epilogue reads neither field
    if (L.save_pre || L.mask.kind != SRC_NONE) {
      ch.layer[l].kind = -1;
      continue;
    }
    // the forecast's output layer: last layer, no activation / norm / addends, n_valid (even) real columns of an N32-row image,
    // output and residual rows 8-byte aligned and not gathered
    const bool narrow = l + 1 == ch.n_layers && L.n_valid < L.N32 && !(L.n_valid & 1) && (L.N32 == 128 || L.N32 == 256) && L.out && !L.relu &&
                        !L.ln_g && !L.feeds_next && !L.seg_dst && L.add[0].kind == SRC_NONE && L.add[1].kind == SRC_NONE &&
                        !(reinterpret_cast<uintptr_t>(L.out) & 7) && !(L.ldo & 1) && L.out_cols >= L.n_valid &&
                        (L.residual.kind == SRC_NONE ||
                         ((L.residual.kind == SRC_STREAM || L.residual.kind == SRC_BCAST) && L.residual.width >= L.n_valid && !(L.residual.ld & 1) &&
                          !(reinterpret_cast<uintptr_t>(L.residual.base + L.residual.col0) & 7) && fits32(L.residual)));
    if (narrow) {
      ch.layer[l].kind = F_NARROW | F_OUT | (L.residual.kind != SRC_NONE ? F_RES : 0);
      ch.fast |= 1 << l;
      continue;
    }
    bool ok = (L.N == 256 || L.N == 128) && L.n_valid == L.N;
    for (int a = 0; a < 2; ++a)
      if (L.add[a].kind != SRC_NONE) ok = ok && src_fast(L.add[a], L.N);
    if (L.residual.kind != SRC_NONE) ok = ok && src_fast(L.residual, L.N);
    if (L.out) ok = ok && aligned32(L.out) && !(L.ldo & 7) && L.out_cols >= L.N;
    if (L.seg_dst) ok = ok && L.seg_out && L.seg_carry && aligned32(L.seg_out) && aligned32(L.seg_carry) && !(L.seg_ld & 7) && L.ln_g && L.N == 256;
    if (L.seg_add) ok = ok && L.seg_dst && aligned32(L.seg_add);
    const int f = (L.add[0].kind != SRC_NONE ? F_ADD0 : 0) | (L.add[1].kind != SRC_NONE ? F_ADD1 : 0) | (L.relu ? F_RELU : 0) |
                  (L.ln_g ? F_LN : 0) | (L.residual.kind != SRC_NONE ? F_RES : 0) | (L.out ? F_OUT : 0) | (L.feeds_next ? F_FEEDS : 0) |
                  (L.seg_dst ? F_SEG : 0);
    bool listed = false;
    if (L.N == 256) {
      for (int k : kinds4) listed = listed || k == f;
    } else {
      for (int k : kinds2) listed = listed || k == f;
    }
    ch.layer[l].kind = listed ? f : -1;
    if (ok && listed) ch.fast |= 1 << l;
  }
}
// Would launch_chain_tc3 run this chain on the lean path?  (gw_forward.cu asks before it decides whether the forecast's 78-column output
// layer rides in the node chain or runs as a general-path chain of its own.)
bool tc3_chain_is_lean(const TcChain& ch_in) {
  TcChain ch = ch_in;
  tc3_mark_lean(ch);
  if (getenv("GW_TC3_NOFAST")) return false;
  const int32_t all = (int32_t)(0x80000000u | ((1u << ch.n_layers) - 1u));
  return ch.fast == all && ch.out_mode == 0;
}
cudaError_t tc_column_block(const TcChain& ch, int n0, int nb, TcChain* out) {
  const TcLayer& L = ch.layer[0];
  if (ch.n_layers != 1 || n0 < 0 || nb <= 0 || nb > TC_COL_BLOCK || n0 + nb > L.n_valid) return cudaErrorInvalidValue;
  if (L.ln_g && (n0 != 0 || nb != L.n_valid)) return cudaErrorInvalidValue;  // a LayerNorm row must stay in one chain
  if (L.feeds_next || L.seg_dst || ch.out_mode != 0) return cudaErrorInvalidValue;
  auto shift = [&](RowSrc s) {  // the source's columns n0 .. n0 + nb - 1
    if (s.kind != SRC_NONE) s.col0 += n0, s.width = std::max(0, std::min(s.width - n0, nb));
    return s;
  };
  *out = ch;
  TcLayer& B = out->layer[0];
  B.Wp = nullptr, B.wamax = nullptr;
  B.N = (nb + 15) / 16 * 16, B.N32 = tc_packed_rows(nb), B.n_valid = nb;
  if (L.bias) B.bias = L.bias + n0;
  for (int a = 0; a < 2; ++a) B.add[a] = shift(L.add[a]);
  B.residual = shift(L.residual), B.mask = shift(L.mask);
  if (L.out) B.out = L.out + n0;
  if (L.save_pre) B.save_pre = L.save_pre + n0;
  B.out_cols = std::max(0, std::min(L.out_cols - n0, nb));
  return cudaSuccess;
}
cudaError_t tc_row_op_chain(const GemmOp& op, TcChain* ch) {
  if (op.add[2].kind != SRC_NONE || op.a[0].kind == SRC_NONE || (op.ln_gamma && op.N > TC_COL_BLOCK)) return cudaErrorInvalidValue;
  *ch = TcChain();
  ch->rows_per_sample = op.rows_per_sample, ch->batch = op.batch;
  ch->a0[0] = op.a[0], ch->a0[1] = op.a[1];
  ch->K0 = (op.K + 63) / 64 * 64, ch->n_layers = 1;
  TcLayer& L = ch->layer[0];
  L.K = ch->K0, L.N = op.N, L.n_valid = op.N;
  L.bias = op.bias, L.add[0] = op.add[0], L.add[1] = op.add[1], L.relu = op.relu;
  L.ln_g = op.ln_gamma, L.ln_b = op.ln_beta, L.residual = op.residual;
  L.out = op.out, L.ldo = op.ldo, L.out_cols = op.N, L.save_pre = op.save_pre, L.mask = op.mask;
  return cudaSuccess;
}
cudaError_t launch_operand_bound(RowSrc& s, int rows_per_sample, int batch, float* amax, cudaStream_t st) {
  if (s.kind != SRC_STREAM && s.kind != SRC_BCAST) return cudaErrorInvalidValue;
  const long long n = (long long)(s.kind == SRC_STREAM ? (long long)batch * s.src_rows : (long long)rows_per_sample) * s.ld;
  const cudaError_t e = launch_absmax_flat(s.base, n, amax, st);
  s.bound = amax, s.bound_mul = 1.f, s.bound_mul_i = nullptr;
  return e;
}
float tc_ln_bound(int N, float gamma_amax, float beta_amax) { return sqrtf((float)N) * gamma_amax + beta_amax; }
cudaError_t launch_chain_tc3(const TcChain& ch_in, cudaStream_t stream) {
  TcChain ch = ch_in;
  using namespace t3;
  static int num_sms[64] = {0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (num_sms[dev] == 0) {
    int n = 0;
    e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    const void* fns[6] = {(const void*)gw_chain_tc3_kernel<true, 0>,  (const void*)gw_chain_tc3_kernel<true, 1>,  (const void*)gw_chain_tc3_kernel<true, 2>,
                          (const void*)gw_chain_tc3_kernel<false, 0>, (const void*)gw_chain_tc3_kernel<false, 1>, (const void*)gw_chain_tc3_kernel<false, 2>};
    for (int i = 0; i < 6; ++i) {
      e = cudaFuncSetAttribute(fns[i], cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
      if (e != cudaSuccess) return e;
    }
    num_sms[dev] = n;
  }
  const long long R = (long long)ch.rows_per_sample * ch.batch;
  if (R <= 0 || ch.n_layers <= 0) return cudaSuccess;
  // structural requirements of the kernel
  if (ch.n_layers > PAR_LAYERS || ch.K0 <= 0 || (ch.K0 & 63)) return cudaErrorInvalidValue;
  int n_ln = 0;
  if (ch.a0[1].kind != SRC_NONE && (ch.a0[0].width & 63)) return cudaErrorInvalidValue;  // a chunk never straddles two sources
  if (ch.layer[ch.n_layers - 1].feeds_next) return cudaErrorInvalidValue;

  for (int l = 0; l < ch.n_layers; ++l) {
    const TcLayer& L = ch.layer[l];
    if (!L.Wp || (L.K & 63) || (L.N & 15) || L.N > 256 || L.N <= 0 || L.n_valid <= 0 || L.n_valid > L.N) return cudaErrorInvalidValue;
    if (L.feeds_next && (L.N & 63)) return cudaErrorInvalidValue;
    if (L.ln_g && L.add[0].kind != SRC_NONE) return cudaErrorInvalidValue;  // addends are applied before ReLU, not before LayerNorm
    // A LayerNorm normalises over the n_valid real columns (ln_stats; the padding columns of the accumulator are exactly zero: zero
    // weight rows and bias).  Padded ones (N = n_valid rounded up to 16) run only as the one-layer chain of a training row op, which
    // takes the general epilogue: its stores, pre-LayerNorm store and residual stop at n_valid columns (out_cols, source widths).
    if (L.ln_g && ((L.n_valid != L.N && ch.n_layers != 1) || ++n_ln > 2)) return cudaErrorInvalidValue;
    if (L.add[0].kind == SRC_NONE && L.add[1].kind != SRC_NONE) return cudaErrorInvalidValue;
    for (int a = 0; a < 2; ++a)
      if (L.add[a].kind != SRC_NONE && L.add[a].kind != SRC_STREAM && L.add[a].kind != SRC_BCAST && L.add[a].kind != SRC_GATHER &&
          L.add[a].kind != SRC_BGATHER)
        return cudaErrorInvalidValue;
    if (L.residual.kind != SRC_NONE && L.residual.kind != SRC_STREAM && L.residual.kind != SRC_BCAST && L.residual.kind != SRC_GATHER &&
        L.residual.kind != SRC_BGATHER)
      return cudaErrorInvalidValue;
    if (L.add[0].kind != SRC_NONE && L.residual.kind != SRC_NONE) return cudaErrorInvalidValue;  // they share the prefetch registers
    if (L.mask.kind != SRC_NONE && L.mask.kind != SRC_STREAM && L.mask.kind != SRC_BCAST && L.mask.kind != SRC_GATHER && L.mask.kind != SRC_BGATHER)
      return cudaErrorInvalidValue;
    if (l == 0 && L.K != ch.K0) return cudaErrorInvalidValue;
    if (l > 0 && !L.reuse_a && (!ch.layer[l - 1].feeds_next || ch.layer[l - 1].N != L.K)) return cudaErrorInvalidValue;
    if (L.reuse_a && (l == 0 || L.K != ch.layer[l - 1].K || ch.layer[l - 1].feeds_next || L.K > 64 * A_SLOTS)) return cudaErrorInvalidValue;  // the whole operand must still be resident
  }
  const int tiles = ((ch.rows_per_sample + TILE_M - 1) / TILE_M) * ch.batch;
  const int grid = tiles < num_sms[dev] ? tiles : num_sms[dev];
  tc3_mark_lean(ch);
  if (getenv("GW_TC3_NOFAST")) ch.fast = 0;
  const int32_t all = (int32_t)(0x80000000u | ((1u << ch.n_layers) - 1u));
  int mode = ch.fast == all ? 1 : 0;
  if (ch.out_mode != 0) mode = 0;  // the multi-GPU boundary stores live in the general path's store tiers
  for (int l = 0; l < ch.n_layers; ++l) {  // both paths run on the perm32 feature order and its row padding (64)
    if (ch.layer[l].N32 < ch.layer[l].N || (ch.layer[l].N32 & 63) || ch.layer[l].N32 > 256) return cudaErrorInvalidValue;
    ch.layer[l].N = ch.layer[l].N32;
  }
  if (mode == 0)
    for (int l = 0; l < ch.n_layers; ++l)
      if (ch.layer[l].seg_dst) return cudaErrorInvalidValue;  // the fused per-target sum exists on the lean path only
  for (int a = 0; a < 2; ++a)
    if (ch.a0[a].kind == SRC_SEGSUM) return cudaErrorInvalidValue;  // reduce with gw_segsum_kernel first (a fused per-thread
                                                                    // reduction in stage 0 was measured slower than the kernel)
#define GW_LAUNCH3(SPLIT_, MODE_) gw_chain_tc3_kernel<SPLIT_, MODE_><<<grid, NUM_THREADS, SMEM_BYTES, stream>>>(ch)
  if (mode == 1 && (ch.layer[ch.n_layers - 1].kind & F_NARROW)) mode = 2;
  if (ch.split) {
    if (mode == 2) GW_LAUNCH3(true, 2); else if (mode == 1) GW_LAUNCH3(true, 1); else GW_LAUNCH3(true, 0);
  } else {
    if (mode == 2) GW_LAUNCH3(false, 2); else if (mode == 1) GW_LAUNCH3(false, 1); else GW_LAUNCH3(false, 0);
  }
#undef GW_LAUNCH3
  count_launch();
  return cudaGetLastError();
}

}  // namespace gw
