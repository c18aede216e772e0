// Warp-specialised bf16 GEMM for sm_90a (one BM x BN output tile per CTA: 128 x 128, 128 x 256 or 192 x 256).
//   warpgroup 0      : TMA producer (cp.async.bulk.tensor 2D / 5D, SWIZZLE_128B, NSTAGE-deep mbarrier ring)
//   warpgroups 1-BM/64: consumers   (wgmma.mma_async m64 x BN x 16 each, fp32 accumulators in registers), then the
//                   epilogue: accumulators staged through shared memory -> each warp along one row, two 4-column quads a thread ->
//                   bias / GELU / GELU' / dropout / residual -> bf16 | fp32 | atomic fp32
// Operands may be K-major or MN-major (the transpose bits of wgmma), so the same kernel serves forward (x.W^T),
// dgrad (dy.W) and wgrad (dy^T.x, split-K with fp32 atomics, or per-slice partials added in slice order in the
// deterministic mode).
#include <cuda.h>

#include <algorithm>

#include "common.h"
#include "philox.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace ymp {

constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int SMEM_OPTIN_MAX = 232448;  // dynamic shared memory a CTA may opt in to on sm_90

struct GemmKParams {
  void* D;
  const __nv_bfloat16* bias;
  const void* residual;            // bf16 or fp32 (res_f32)
  __nv_bfloat16* aux_out;
  const __nv_bfloat16* aux_in;
  int M, N, K;
  int ldd, ldr;
  int a_mn, b_mn;
  int act, out_f32, accumulate, split_k;
  int kb_per_split;
  int res_row_mod;                 // residual row = row % res_row_mod (0: plain)
  int d_row_block, d_row_stride;   // D row = (row / block) * stride + row % block (0: plain)
  int res_f32;
  int n_fast;                      // tile order: consecutive units walk N first (A streamed once) or M first
  float alpha;
  int im2col_T, im2col_N, im2col_Wp;  // fused im2col A operand (im2col_T > 0): frames, patches per frame, patches per row
  DropSpec drop;                   // dropout before the residual add (has_drop)
  int has_drop;
};

// BM = 192 exists for BN = 256 only: it brings (192 + 256) operand bytes per 192 x 256 k-block product against
// (128 + 256) per 128 x 256, 22 % fewer L2 bytes per FLOP, and its epilogue runs on 384 threads instead of 256.  It has
// no producer warpgroup: ptxas compiles every instruction within the register count the launch bounds leave (128 at
// 512 threads, whatever setmaxnreg does at run time), and one m64n256 wgmma alone needs 154.  So its three consumer
// warpgroups are the whole CTA (384 threads, 168 registers, as for BM = 128), and thread 0 refills the ring.
template <int BM, int BN>
struct GemmCfg {
  static_assert((BM == 128 && (BN == 128 || BN == 256)) || (BM == 192 && BN == 256), "tile shapes");
  static constexpr int CONSUMERS = BM / 64;             // consumer warpgroups, 64 rows each
  static constexpr bool PRODUCER_WG = CONSUMERS == 2;   // warpgroup 0 is a TMA producer
  static constexpr int THREADS = 128 * (CONSUMERS + PRODUCER_WG);
  static constexpr int FIRST_CONSUMER = THREADS - 128 * CONSUMERS;
  static constexpr int NSTAGE = (BN == 256) ? 4 : 6;    // 192 KB operand ring for BM = 128, 224 KB for 192
  static constexpr int A_STAGE_BYTES = BM * BK * 2;
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STG_LD = BN + 4;                 // fp32 staging row (+4: conflict-free row-per-thread reads)
  static_assert(BM * STG_LD * 4 <= NSTAGE * STAGE_BYTES, "epilogue staging reuses the operand ring");
  static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + 256 + 1024;
  static_assert(SMEM_BYTES <= SMEM_OPTIN_MAX, "ring, barriers and alignment pad fit the opt-in shared memory");
};

// Epilogue thread layout: the threads of a warp cover consecutive columns of one output row (two rows for BN = 128), so
// every global access of the epilogue is coalesced along the row and every staging read is a contiguous run of shared
// memory.  A thread owns two 4-column quads of the tile, columns 4j .. 4j+3 and BN/2 + 4j .. +3, in every RPP-th row;
// its bias is loaded once.
template <int BM, int BN>
struct EpiCfg {
  static constexpr int THREADS = 2 * BM;    // the consumer warpgroups
  static constexpr int TPR = BN / 8;        // threads per row
  static constexpr int RPP = THREADS / TPR; // rows per pass of the epilogue threads
  static constexpr int GROUP = 4;           // rows whose global operands are fetched together
  static_assert(BM % (RPP * GROUP) == 0, "row groups tile BM");
};

// bf16 quad (8 bytes) <-> 4 floats
__device__ __forceinline__ uint2 ld_bf16x4(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const uint2*>(p)); }
__device__ __forceinline__ void st_bf16x4(__nv_bfloat16* p, const float* f) {
  *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]));
}

// The epilogue's flags are uniform over a launch, but tested per row they are some fifty branches, most of them taken,
// and with two warps per scheduler nothing hides them: the row loop of a plain bf16 tile took 10 500 cycles, with or
// without its stores.  So the row loop is compiled once per flag combination the training step launches (KIND >= 0:
// the flags below are constants and the untaken code is gone) and once with every flag read at run time (EPI_ANY),
// which serves everything else (dropout, an activation without act', bf16 residual, ...).  Same statements, same
// order: the results are bit-identical whichever copy runs.
constexpr int EPI_ANY = -1;
enum { EPI_AUX_NONE = 0, EPI_AUX_MUL = 1, EPI_AUX_GELU_ERF = 2, EPI_AUX_GELU_TANH = 3 };  // 2, 3: act' stored in aux_out
enum { EPI_OUT_BF16 = 0, EPI_OUT_F32 = 1, EPI_OUT_ATOMIC = 2 };
constexpr int epi_kind(int aux, int res_f32, int out) { return aux * 16 + res_f32 * 4 + out; }
template <int KIND>
struct EpiFlags {
  bool aux_in, aux_out, residual, res_f32, out_f32, accumulate;
  int act;
  __device__ __forceinline__ explicit EpiFlags(const GemmKParams& p) {
    if constexpr (KIND == EPI_ANY) {
      aux_in = p.aux_in != nullptr; aux_out = p.aux_out != nullptr; act = p.act;
      residual = p.residual != nullptr; res_f32 = p.res_f32 != 0;
      out_f32 = p.out_f32 != 0; accumulate = p.accumulate != 0;
    } else {
      constexpr int aux = KIND / 16, out = KIND % 4;
      aux_in = aux == EPI_AUX_MUL; aux_out = aux >= EPI_AUX_GELU_ERF;
      act = aux == EPI_AUX_GELU_ERF ? YMP_ACT_GELU_ERF : aux == EPI_AUX_GELU_TANH ? YMP_ACT_GELU_TANH : YMP_ACT_NONE;
      residual = res_f32 = (KIND / 4) % 4 != 0;
      out_f32 = out != EPI_OUT_BF16; accumulate = out == EPI_OUT_ATOMIC;
    }
  }
};
// The combination of a launch, or EPI_ANY when no specialised copy exists for it.
__device__ __forceinline__ int epi_kind_of(const GemmKParams& p) {
  const int aux = p.aux_in ? EPI_AUX_MUL
                  : (p.act == YMP_ACT_NONE && !p.aux_out) ? EPI_AUX_NONE
                  : (p.act == YMP_ACT_GELU_ERF && p.aux_out) ? EPI_AUX_GELU_ERF
                  : (p.act == YMP_ACT_GELU_TANH && p.aux_out) ? EPI_AUX_GELU_TANH : -1;
  if (aux < 0 || p.has_drop || (p.residual && !p.res_f32)) return EPI_ANY;
  return epi_kind(aux, p.residual ? 1 : 0, !p.out_f32 ? EPI_OUT_BF16 : p.accumulate ? EPI_OUT_ATOMIC : EPI_OUT_F32);
}

// Global operands of one row of a thread's two quads, fetched for a group of rows before any of them is stored.
struct EpiIn {
  uint32_t res[8];  // 8 fp32, or 8 bf16 in the first 4 words
  uint32_t aux[4];  // 8 bf16 (aux_in)
};
template <int KIND>
__device__ __forceinline__ void epilogue_fetch(const GemmKParams& p, int row, const int (&col)[2], bool full, EpiIn& in) {
  const EpiFlags<KIND> f(p);
  if (row >= p.M || !full) return;
  if (f.aux_in) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const uint2 a = ld_bf16x4(p.aux_in + (size_t)row * p.ldd + col[q]);
      in.aux[2 * q] = a.x; in.aux[2 * q + 1] = a.y;
    }
  }
  if (f.residual) {
    const int rrow = p.res_row_mod ? row % p.res_row_mod : row;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (f.res_f32) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.residual) + (size_t)rrow * p.ldr + col[q]));
        in.res[4 * q] = __float_as_uint(a.x); in.res[4 * q + 1] = __float_as_uint(a.y);
        in.res[4 * q + 2] = __float_as_uint(a.z); in.res[4 * q + 3] = __float_as_uint(a.w);
      } else {
        const uint2 a = ld_bf16x4(reinterpret_cast<const __nv_bfloat16*>(p.residual) + (size_t)rrow * p.ldr + col[q]);
        in.res[2 * q] = a.x; in.res[2 * q + 1] = a.y;
      }
    }
  }
}

// Epilogue of one row of a thread's two quads: v[4q + e] is column col[q] + e.  `full`: both quads lie inside N.
template <bool DROP, int KIND>
__device__ __forceinline__ void epilogue_row(const GemmKParams& p, float (&v)[8], int row, const int (&col)[2], bool full,
                                             const uint32_t (&bias)[4], const EpiIn& in, const DropState& ds) {
  if (row >= p.M) return;
  const EpiFlags<KIND> f(p);
  const int drow = p.d_row_block ? (row / p.d_row_block) * p.d_row_stride + row % p.d_row_block : row;
  const int rrow = p.res_row_mod ? row % p.res_row_mod : row;
  if (p.alpha != 1.0f) {
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = v[i] * p.alpha;
  }

  if (full) {
    if (p.bias) {
#pragma unroll
      for (int i = 0; i < 4; ++i) { v[2 * i] += bf16_lo(bias[i]); v[2 * i + 1] += bf16_hi(bias[i]); }
    }
    const size_t off[2] = {(size_t)row * p.ldd + col[0], (size_t)row * p.ldd + col[1]};      // aux tensors: plain rows
    const size_t doff[2] = {(size_t)drow * p.ldd + col[0], (size_t)drow * p.ldd + col[1]};   // D: optionally re-blocked
    // aux_out: with an activation it receives act'(v) (what the backward epilogue multiplies by),
    // without one the value itself.  aux_in: a plain multiplier.  Switches are warp-uniform.
    if (f.aux_in) {
#pragma unroll
      for (int i = 0; i < 4; ++i) { v[2 * i] *= bf16_lo(in.aux[i]); v[2 * i + 1] *= bf16_hi(in.aux[i]); }
    } else if (f.act == YMP_ACT_GELU_ERF) {
      if (f.aux_out) {
        float x[8], d[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = v[i];
        gelu_erf_both_x8(x, v, d);
        st_bf16x4(p.aux_out + off[0], d);
        st_bf16x4(p.aux_out + off[1], d + 4);
      } else {
        float x[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) x[i] = v[i];
        gelu_erf_x8(x, v);
      }
    } else if (f.act == YMP_ACT_GELU_TANH) {
      if (f.aux_out) {
        float d[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = gelu_tanh_both(v[i], d[i]);
        st_bf16x4(p.aux_out + off[0], d);
        st_bf16x4(p.aux_out + off[1], d + 4);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = gelu_tanh(v[i]);
      }
    } else if (f.aux_out) {
      st_bf16x4(p.aux_out + off[0], v);
      st_bf16x4(p.aux_out + off[1], v + 4);
    }
    if constexpr (DROP) {  // bias-dropout-add: residual + dropout(x + bias)
#pragma unroll
      for (int q = 0; q < 2; ++q) drop4(ds, (uint32_t)row, (uint32_t)col[q], v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
    if (f.residual) {
      if (f.res_f32) {  // fp32 residual stream
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] += __uint_as_float(in.res[i]);
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) { v[2 * i] += bf16_lo(in.res[i]); v[2 * i + 1] += bf16_hi(in.res[i]); }
      }
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      if (!f.out_f32) {
        st_bf16x4(reinterpret_cast<__nv_bfloat16*>(p.D) + doff[q], v + 4 * q);
      } else if (!f.accumulate) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.D) + doff[q]) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
      } else {
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(reinterpret_cast<float*>(p.D) + doff[q]),
                     "f"(v[4 * q]), "f"(v[4 * q + 1]), "f"(v[4 * q + 2]), "f"(v[4 * q + 3])
                     : "memory");
      }
    }
  } else {
    // ragged N tail: scalar, bounds-checked
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = col[i >> 2] + (i & 3);
      if (c < p.N) {
        float x = v[i];
        if (p.bias) x += __bfloat162float(p.bias[c]);
        const size_t off = (size_t)row * p.ldd + c, doff = (size_t)drow * p.ldd + c;
        if (f.aux_in) {
          x *= __bfloat162float(p.aux_in[off]);
        } else if (f.act == YMP_ACT_GELU_ERF) {
          float d; x = gelu_erf_both(x, d);
          if (f.aux_out) p.aux_out[off] = __float2bfloat16(d);
        } else if (f.act == YMP_ACT_GELU_TANH) {
          float d; x = gelu_tanh_both(x, d);
          if (f.aux_out) p.aux_out[off] = __float2bfloat16(d);
        } else if (f.aux_out) {
          p.aux_out[off] = __float2bfloat16(x);
        }
        if constexpr (DROP) {
          const uint4 w = drop_words(ds, (uint32_t)row, (uint32_t)c >> 2);
          const uint32_t wc = (c & 3) == 0 ? w.x : (c & 3) == 1 ? w.y : (c & 3) == 2 ? w.z : w.w;
          x = wc >= ds.thresh ? x * ds.scale : 0.f;
        }
        if (f.residual)
          x += f.res_f32 ? reinterpret_cast<const float*>(p.residual)[(size_t)rrow * p.ldr + c]
                         : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.residual)[(size_t)rrow * p.ldr + c]);
        if (!f.out_f32) reinterpret_cast<__nv_bfloat16*>(p.D)[doff] = __float2bfloat16(x);
        else if (!f.accumulate) reinterpret_cast<float*>(p.D)[doff] = x;
        else atomicAdd(reinterpret_cast<float*>(p.D) + doff, x);
      }
    }
  }
}

// ---------------------------------------------------------------- fused im2col A operand (patch embedding)
// One 128-row x 64-column tile of the implicit patch matrix (rows m0 .. m0+127 = 128/T consecutive patches x T frames,
// columns kb*64 .. +63 = 4 pixel rows x 16 pixels of one channel) arrives as FOUR 16-column sub-tiles of 4 KB, one per
// pixel row: every patch contributes one 5-D box {16 px, 1 row, T frames} = T rows x 32 bytes, which with
// SWIZZLE_32B is exactly T/8 shared-memory atoms of 8 rows x 32 bytes, dense (a 128-byte-swizzled box would give every
// 32-byte line its own 128-byte row).  Each sub-tile is the A operand of one wgmma K-step
// (K = 16) through a SWIZZLE_32B descriptor; rows past the last sample are out of range and arrive as zeros.
// Only the 128-row tiles take it.
constexpr int IM2COL_BM = 128;
constexpr int IM2COL_SUB_BYTES = IM2COL_BM * 32;  // one 128-row x 16-column sub-tile
__device__ __forceinline__ void load_a_im2col(uint8_t* sa, const CUtensorMap* tma, uint64_t* bar, int m0, int kb,
                                              const GemmKParams& p) {
  const int T = p.im2col_T, c = kb >> 2, y0 = (kb & 3) * 4;
  const int pt = m0 / T;  // first patch (global index b*N + n) of the tile
  for (int i = 0; i < IM2COL_BM / T; ++i) {
    const int g = pt + i, b = g / p.im2col_N, n = g - b * p.im2col_N;
    const int ny = n / p.im2col_Wp, nx = n - ny * p.im2col_Wp;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      uint8_t* dst = sa + ks * IM2COL_SUB_BYTES + i * T * 32;
      tma_load_5d(dst, tma, bar, nx * 16, ny * 16 + y0 + ks, 0, c, b);
    }
  }
}
// ---------------------------------------------------------------- kernel
// Accumulator fragment of wgmma m64nBN (thread t of a consumer warpgroup): acc[4j + e] holds row 16 (t / 32) + (t % 32) / 4
// (+8 for e >= 2), column 8 j + 2 (t % 4) + (e & 1) of the warpgroup's 64-row slice.
__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// The row loop of the epilogue over the staged tile, for one flag combination (see EpiFlags).
template <int BM, int BN, int KIND>
__device__ __forceinline__ void epilogue_rows(const GemmKParams& p, const float* stg, int m_blk, int n_blk) {
  using Cfg = GemmCfg<BM, BN>;
  using Epi = EpiCfg<BM, BN>;
  DropState ds;  // only read when has_drop
  if (KIND == EPI_ANY && p.has_drop) ds = drop_state(p.drop);
  const int et = threadIdx.x - Cfg::FIRST_CONSUMER, tj = et % Epi::TPR, tr = et / Epi::TPR;
  const int col[2] = {n_blk * BN + 4 * tj, n_blk * BN + BN / 2 + 4 * tj};
  const bool full = col[1] + 4 <= p.N;
  uint32_t bias[4];
  if (p.bias && full) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const uint2 b = ld_bf16x4(p.bias + col[q]);
      bias[2 * q] = b.x; bias[2 * q + 1] = b.y;
    }
  }
#pragma unroll 1
  for (int lr0 = tr; lr0 < BM; lr0 += Epi::RPP * Epi::GROUP) {
    EpiIn in[Epi::GROUP];
#pragma unroll
    for (int u = 0; u < Epi::GROUP; ++u) epilogue_fetch<KIND>(p, m_blk * BM + lr0 + u * Epi::RPP, col, full, in[u]);
#pragma unroll
    for (int u = 0; u < Epi::GROUP; ++u) {
      const int lr = lr0 + u * Epi::RPP;
      const float4 a = *reinterpret_cast<const float4*>(stg + lr * Cfg::STG_LD + 4 * tj);
      const float4 b = *reinterpret_cast<const float4*>(stg + lr * Cfg::STG_LD + BN / 2 + 4 * tj);
      float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      if (KIND == EPI_ANY && p.has_drop) epilogue_row<true, KIND>(p, v, m_blk * BM + lr, col, full, bias, in[u], ds);
      else epilogue_row<false, KIND>(p, v, m_blk * BM + lr, col, full, bias, in[u], ds);
    }
  }
}

// One CTA: the tile's K range [kb0, kb1) of slice ks, then the epilogue.  PARTIAL (deterministic split-K): the
// alpha-scaled fp32 tile is stored, without any other epilogue step, to slice ks of the workspace p.D ([split_k, M,
// ldd]); ordered_sum then adds the slices to D in slice order.
template <int BM, int BN, int AMN, int BMN, bool PARTIAL>
__device__ __forceinline__ void gemm_tile(const CUtensorMap& tma_a, const CUtensorMap& tma_b, const GemmKParams& p) {
  using Cfg = GemmCfg<BM, BN>;
  constexpr int NSTAGE = Cfg::NSTAGE;
  constexpr int A_STAGE_BYTES = Cfg::A_STAGE_BYTES;
  constexpr bool IM2COL = BM == IM2COL_BM;  // the fused im2col operand can occur (p.im2col_T decides)
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment in the shared address space
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + NSTAGE * A_STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + NSTAGE * Cfg::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + NSTAGE;

  const int wg = threadIdx.x >> 7;
  const int num_m = (p.M + BM - 1) / BM;
  const int num_n = (p.N + BN - 1) / BN;
  const int kb_total = (p.K + BK - 1) / BK;
  const int ks = blockIdx.x % p.split_k;
  const int t = blockIdx.x / p.split_k;
  const int m_blk = p.n_fast ? t / num_n : t % num_m;
  const int n_blk = p.n_fast ? t % num_n : t / num_m;
  const int kb0 = ks * p.kb_per_split;
  const int kb1 = min(kb_total, kb0 + p.kb_per_split);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int i = 0; i < NSTAGE; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], Cfg::CONSUMERS);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  // k-block kb into ring slot `stage`, completion on its full barrier
  auto load_stage = [&](int kb, int stage) {
    mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
    uint8_t* sa = smem_a + stage * A_STAGE_BYTES;
    uint8_t* sb = smem_b + stage * Cfg::B_STAGE_BYTES;
    if (IM2COL && p.im2col_T) {
      load_a_im2col(sa, &tma_a, &full_bar[stage], m_blk * BM, kb, p);
    } else if (!AMN) {
      tma_load_2d(sa, &tma_a, &full_bar[stage], kb * BK, m_blk * BM);
    } else {
#pragma unroll
      for (int c = 0; c < BM / 64; ++c)
        tma_load_2d(sa + c * (64 * BK * 2), &tma_a, &full_bar[stage], m_blk * BM + c * 64, kb * BK);
    }
    if (!BMN) {
      tma_load_2d(sb, &tma_b, &full_bar[stage], kb * BK, n_blk * BN);
    } else {
#pragma unroll
      for (int c = 0; c < BN / 64; ++c)
        tma_load_2d(sb + c * (64 * BK * 2), &tma_b, &full_bar[stage], n_blk * BN + c * 64, kb * BK);
    }
  };

  if constexpr (Cfg::PRODUCER_WG) {
    if (wg == 0) {
      // =================================================================== TMA producer
      if (threadIdx.x == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          load_stage(kb, stage);
          if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
        }
      }
      return;
    }
  } else if (threadIdx.x == 0) {
    // no producer warpgroup: the empty ring is filled here, and refilled slot by slot in the main loop
    for (int i = 0; i < NSTAGE && kb0 + i < kb1; ++i) load_stage(kb0 + i, i);
  }

  // ======================================================================= consumers: rows 64 cw .. +63
  const int cw = wg - Cfg::PRODUCER_WG;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  // K-major: rows of 128 B, 8-row swizzle atoms 1024 B apart (SBO); a K step of 16 is 32 B along the row.
  // MN-major: 64-element (128 B) MN chunks of 64 k-rows = 8192 B apart (LBO); 8-k-row groups 1024 B apart (SBO);
  //           a K step of 16 is two groups.  Either way the warpgroup's 64-row slice of A starts 8192 B in.
  // Fused im2col A: SWIZZLE_32B sub-tiles of 128 rows x 16 columns (4096 B), 8-row atoms 256 B apart.
  {
    int stage = 0;
    uint32_t phase = 0;
    int prev = -1;
    wgmma_fence_acc(acc);
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem_a + stage * A_STAGE_BYTES);
      const uint32_t sb = smem_u32(smem_b + stage * Cfg::B_STAGE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WGMMA_K; ++k) {
        const uint64_t da = IM2COL && p.im2col_T ? make_smem_desc(sa + k * IM2COL_SUB_BYTES + cw * 64 * 32, 16, 256, 3)
                            : AMN ? make_smem_desc(sa + cw * 8192 + k * WGMMA_K * 128, 64 * BK * 2, 1024, 1)
                                  : make_smem_desc(sa + cw * 8192 + k * WGMMA_K * 2, 16, 1024, 1);
        const uint64_t db = BMN ? make_smem_desc(sb + k * WGMMA_K * 128, 64 * BK * 2, 1024, 1)
                                : make_smem_desc(sb + k * WGMMA_K * 2, 16, 1024, 1);
        if constexpr (BN == 256) wgmma_m64n256<AMN, BMN>(acc, da, db, 1u);
        else wgmma_m64n128<AMN, BMN>(acc, da, db, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs have retired: its slot may be refilled
      if (prev >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev]);
      if constexpr (!Cfg::PRODUCER_WG) {
        // k-block kb - 1 + NSTAGE takes the previous k-block's slot once every warpgroup has released it (release
        // number (kb - 1 - kb0) / NSTAGE of that slot)
        if (threadIdx.x == 0 && prev >= 0 && kb - 1 + NSTAGE < kb1) {
          mbar_wait(&empty_bar[prev], ((kb - 1 - kb0) / NSTAGE) & 1);
          load_stage(kb - 1 + NSTAGE, prev);
        }
      }
      prev = stage;
      if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
  }

  // ======================================================================= epilogue
  // Every operand byte has been consumed (the ring holds this tile only), so the ring becomes the fp32 staging tile.
  named_sync(1, 128 * Cfg::CONSUMERS);
  float* stg = reinterpret_cast<float*>(smem);
  {
    const int lt = threadIdx.x & 127, r0 = cw * 64 + (lt >> 5) * 16 + ((lt & 31) >> 2), c0 = 2 * (lt & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(stg + r0 * Cfg::STG_LD + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + (r0 + 8) * Cfg::STG_LD + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  named_sync(1, 128 * Cfg::CONSUMERS);
  if constexpr (PARTIAL) {
    GemmKParams q = p;
    q.D = reinterpret_cast<float*>(p.D) + (size_t)ks * p.M * p.ldd;
    epilogue_rows<BM, BN, epi_kind(EPI_AUX_NONE, 0, EPI_OUT_F32)>(q, stg, m_blk, n_blk);
    return;
  }
  switch (epi_kind_of(p)) {  // uniform over the launch
#define YMP_EPI_CASE(aux, res, out) \
    case epi_kind(aux, res, out): epilogue_rows<BM, BN, epi_kind(aux, res, out)>(p, stg, m_blk, n_blk); break;
    YMP_EPI_CASE(EPI_AUX_NONE, 0, EPI_OUT_BF16)        // qkv, dgrads, LM head
    YMP_EPI_CASE(EPI_AUX_NONE, 1, EPI_OUT_F32)         // projections onto the fp32 residual stream
    YMP_EPI_CASE(EPI_AUX_NONE, 0, EPI_OUT_ATOMIC)      // wgrad
    YMP_EPI_CASE(EPI_AUX_GELU_ERF, 0, EPI_OUT_BF16)    // ViT fc1
    YMP_EPI_CASE(EPI_AUX_GELU_TANH, 0, EPI_OUT_BF16)   // GPT h->4h
    YMP_EPI_CASE(EPI_AUX_MUL, 0, EPI_OUT_BF16)         // their dgrads
#undef YMP_EPI_CASE
    default: epilogue_rows<BM, BN, EPI_ANY>(p, stg, m_blk, n_blk);
  }
}

template <int BM, int BN, int AMN, int BMN>
__global__ void __launch_bounds__(GemmCfg<BM, BN>::THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                       const GemmKParams p) {
  gemm_tile<BM, BN, AMN, BMN, false>(tma_a, tma_b, p);
}

template <int BM, int BN, int AMN, int BMN>
__global__ void __launch_bounds__(GemmCfg<BM, BN>::THREADS, 1)
gemm_bf16_wgmma_partial_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                               const GemmKParams p) {
  gemm_tile<BM, BN, AMN, BMN, true>(tma_a, tma_b, p);
}

// ------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(f);
    else
      cudaGetLastError();
  }
  return fn;
}

// 2D bf16 tensor map: inner (contiguous) extent `inner`, `outer` rows of stride ld elements.
static int make_map(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld,
                    uint32_t box_inner, uint32_t box_outer) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(YMP_ECUDA, "cuTensorMapEncodeTiled entry point unavailable (no driver?)");
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(YMP_ECUDA, "cuTensorMapEncodeTiled failed (%d): inner=%llu outer=%llu ld=%llu",
                     (int)r, (unsigned long long)inner, (unsigned long long)outer,
                     (unsigned long long)ld);
  return YMP_OK;
}

// 5D map over a bf16 video [B, C, T, H, W] for the fused im2col A operand: box {16 px, 1 row, T frames, 1, 1}, SWIZZLE_32B
static int make_video_map(CUtensorMap* m, const ymp_gemm_args* a) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error(YMP_ECUDA, "cuTensorMapEncodeTiled entry point unavailable (no driver?)");
  const cuuint64_t W = a->im2col_W, H = a->im2col_H, T = a->im2col_T, C = a->im2col_C, B = a->im2col_B;
  cuuint64_t dims[5] = {W, H, T, C, B};
  cuuint64_t strides[4] = {W * 2, H * W * 2, T * H * W * 2, C * T * H * W * 2};
  cuuint32_t box[5] = {16, 1, (cuuint32_t)T, 1, 1};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(a->A), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(YMP_ECUDA, "cuTensorMapEncodeTiled (video, 5-D) failed (%d)", (int)r);
  return YMP_OK;
}

template <int BM, int BN, int AMN, int BMN, bool PARTIAL>
static int launch_gemm_t(const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& kp, int grid, cudaStream_t stream) {
  using Cfg = GemmCfg<BM, BN>;
  constexpr auto kernel = PARTIAL ? gemm_bf16_wgmma_partial_kernel<BM, BN, AMN, BMN> : gemm_bf16_wgmma_kernel<BM, BN, AMN, BMN>;
  static DeviceOnce once;
  if (once.first())
    YMP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
  kernel<<<grid, Cfg::THREADS, Cfg::SMEM_BYTES, stream>>>(ta, tb, kp);
  YMP_LAUNCH_CHECK();
  return YMP_OK;
}

template <int BM, int BN, bool PARTIAL = false>
static int launch_gemm(const ymp_gemm_args* a, const GemmKParams& kp, cudaStream_t stream) {
  CUtensorMap ta, tb;
  int rc;
  if (a->im2col_P) rc = make_video_map(&ta, a);
  else if (!a->a_mn_major) rc = make_map(&ta, a->A, a->K, a->M, a->lda, BK, BM);
  else rc = make_map(&ta, a->A, a->M, a->K, a->lda, 64, BK);
  if (rc) return rc;
  if (!a->b_mn_major) rc = make_map(&tb, a->B, a->K, a->N, a->ldb, BK, BN);
  else rc = make_map(&tb, a->B, a->N, a->K, a->ldb, 64, BK);
  if (rc) return rc;
  const int num_m = (a->M + BM - 1) / BM, num_n = (a->N + BN - 1) / BN;
  const int grid = num_m * num_n * kp.split_k;
  switch (kp.a_mn * 2 + kp.b_mn) {
    case 0: return launch_gemm_t<BM, BN, 0, 0, PARTIAL>(ta, tb, kp, grid, stream);
    case 1: return launch_gemm_t<BM, BN, 0, 1, PARTIAL>(ta, tb, kp, grid, stream);
    case 2: return launch_gemm_t<BM, BN, 1, 0, PARTIAL>(ta, tb, kp, grid, stream);
    default: return launch_gemm_t<BM, BN, 1, 1, PARTIAL>(ta, tb, kp, grid, stream);
  }
}

// What one CTA per SM spends on a tile, in µs: t per 64-deep k-block of MMAs, f whatever the tile's K (ring fill,
// epilogue, turnover), f_acc the same with the fp32-atomic epilogue of split-K.  Fitted by tools/gemm_tile_cost.py
// (DESIGN.md §5) on an H100 80GB HBM3 at 700 W; only their ratios matter for the choices below.
struct TileCost { double t, f, f_acc; };
constexpr TileCost TILE_COST_128 = {0.78, 5.0, 14.7};   // 128 x 256
constexpr TileCost TILE_COST_192 = {1.09, 8.0, 20.0};   // 192 x 256

// A launch of `tiles` output tiles, kb_total k-blocks deep, as waves of one tile per SM: µs of a K split count `split`,
// or with split = 0 the count the cost model picks (1 unless accumulating: the K splits then add into D).
struct GemmPlan { int split; double us; };
static GemmPlan plan_gemm(long tiles, int kb_total, int split, bool accumulate, int sms, const TileCost& c) {
  auto cost = [&](int sp) {
    const long waves = (tiles * sp + sms - 1) / sms;
    return waves * (((kb_total + sp - 1) / sp) * c.t + (accumulate ? c.f_acc : c.f));
  };
  if (split > 0) return {split, cost(std::min(split, kb_total))};
  GemmPlan best{1, cost(1)};
  if (accumulate) {
    for (int sp = 2; sp <= 64 && sp * 8 <= kb_total; ++sp) {
      const double us = cost(sp);
      if (us < best.us) best = {sp, us};
    }
  }
  return best;
}

// Checks, plans and launches one GEMM; with ws_bytes set it only reports the workspace the launch needs (bytes of the
// deterministic split-K partials, 0 when the mode is off or the plan has one K slice) and launches nothing.
static int gemm_run(const ymp_gemm_args* a, int tile_m, void* workspace, void* stream, int64_t* ws_bytes) {
  YMP_CHECK_ARG(a != nullptr, "ymp_gemm: null args");
  YMP_CHECK_ARG(a->A && a->B && a->D, "ymp_gemm: null A/B/D");
  YMP_CHECK_ARG(a->M > 0 && a->N > 0 && a->K > 0, "ymp_gemm: bad shape M=%d N=%d K=%d", a->M, a->N, a->K);
  if (a->im2col_P) {
    const int P = a->im2col_P, T = a->im2col_T;
    YMP_CHECK_ARG(P == 16 && T > 0 && T % 8 == 0 && 128 % T == 0 && a->im2col_H % P == 0 && a->im2col_W % P == 0 && !a->a_mn_major,
                  "ymp_gemm(im2col): needs P = 16, T %% 8 == 0, 128 %% T == 0, H, W multiples of P (P=%d T=%d H=%d W=%d)", P, T,
                  a->im2col_H, a->im2col_W);
    const long rows = (long)a->im2col_B * (a->im2col_H / P) * (a->im2col_W / P) * T;
    YMP_CHECK_ARG(a->M == rows && a->K == a->im2col_C * P * P, "ymp_gemm(im2col): needs M = B*N*T, K = C*P*P (M=%d K=%d)", a->M, a->K);
  }
  const bool ia = a->im2col_P != 0;
  YMP_CHECK_ARG((ia || a->lda % 8 == 0) && a->ldb % 8 == 0, "ymp_gemm: lda/ldb must be multiples of 8 (lda=%d ldb=%d)", a->lda, a->ldb);
  YMP_CHECK_ARG(aligned16(a->A) && aligned16(a->B) && aligned16(a->D), "ymp_gemm: A/B/D must be 16-byte aligned");
  YMP_CHECK_ARG(ia || a->lda >= (a->a_mn_major ? a->M : a->K), "ymp_gemm: lda too small");
  YMP_CHECK_ARG(a->ldb >= (a->b_mn_major ? a->N : a->K), "ymp_gemm: ldb too small");
  YMP_CHECK_ARG(a->ldd >= a->N && a->ldd % 8 == 0, "ymp_gemm: ldd must be >= N and a multiple of 8 (ldd=%d)", a->ldd);
  YMP_CHECK_ARG(a->act >= 0 && a->act <= 2, "ymp_gemm: bad act %d", a->act);
  YMP_CHECK_ARG(!a->residual || (a->ldr >= a->N && a->ldr % 8 == 0 && aligned16(a->residual)), "ymp_gemm: bad residual ld/alignment");
  YMP_CHECK_ARG(a->residual_dtype == YMP_DT_BF16 || a->residual_dtype == YMP_DT_F32, "ymp_gemm: bad residual_dtype");
  YMP_CHECK_ARG(!a->bias || aligned16(a->bias), "ymp_gemm: bias must be 16-byte aligned");
  YMP_CHECK_ARG(!a->aux_out || aligned16(a->aux_out), "ymp_gemm: aux_out alignment");
  YMP_CHECK_ARG(!a->aux_in || aligned16(a->aux_in), "ymp_gemm: aux_in alignment");
  YMP_CHECK_ARG(!(a->accumulate && a->out_dtype != YMP_DT_F32), "ymp_gemm: accumulate needs fp32 output");
  // every K-split's epilogue adds its partial to D, so a bias would be added once per split
  YMP_CHECK_ARG(!(a->accumulate && (a->bias || a->aux_out || a->aux_in || a->act || a->residual)),
                "ymp_gemm: accumulate mode supports only alpha and bias-free linear epilogue");
  YMP_CHECK_ARG(a->res_row_mod >= 0 && a->d_row_block >= 0 && (a->d_row_block == 0 || a->d_row_stride >= a->d_row_block),
                "ymp_gemm: bad res_row_mod / d_row_block / d_row_stride");
  YMP_CHECK_ARG(!(a->drop.rng && a->drop.p > 0.f) || (a->drop.p < 1.f && !a->aux_out && !a->accumulate),
                "ymp_gemm: dropout needs 0 < p < 1 and is not combined with aux_out / accumulate");
  YMP_CHECK_ARG(a->tile_n == 0 || a->tile_n == 128 || a->tile_n == 256 || a->tile_n == 512,
                "ymp_gemm: tile_n must be 0 (auto), 128, 256 or 512 (the widest tile: 256 columns on sm_90)");
  YMP_CHECK_ARG(tile_m == 0 || tile_m == 128 || tile_m == 192, "ymp_gemm: tile_m must be 0 (auto), 128 or 192 (tile_m=%d)", tile_m);
  YMP_CHECK_ARG(tile_m != 192 || (a->tile_n != 128 && !a->im2col_P),
                "ymp_gemm: tile_m = 192 needs the 256-column tile and no fused im2col operand");

  const int kb_total = (a->K + BK - 1) / BK;
  const int sms = num_sms();
  int bn = a->tile_n == 512 ? 256 : a->tile_n;
  if (tile_m == 192) bn = 256;
  if (a->im2col_P && bn == 0) bn = (a->N <= 128) ? 128 : 256;
  if (bn == 0) {
    // the 128x256 tile when it fills the machine (or for split-K accumulation); 128x128 when N is narrow or the
    // wide tile would leave SMs idle
    const long t256 = (long)((a->M + 127) / 128) * ((a->N + 255) / 256);
    bn = (a->N <= 128 || (t256 < sms && a->split_k <= 1 && !a->accumulate)) ? 128 : 256;
  }
  // 192 rows when the 256-column tile runs and the cost model puts it below 128 rows: fewer operand bytes per FLOP and
  // epilogue threads per row, against coarser waves and more rows past M
  const bool acc = a->accumulate != 0;
  const long tiles128 = (long)((a->M + 127) / 128) * ((a->N + bn - 1) / bn);
  GemmPlan plan = plan_gemm(tiles128, kb_total, a->split_k, acc, sms, TILE_COST_128);
  int bm = 128;
  if (tile_m == 192 || (tile_m == 0 && bn == 256 && !a->im2col_P)) {
    const GemmPlan p192 = plan_gemm((long)((a->M + 191) / 192) * ((a->N + 255) / 256), kb_total, a->split_k, acc, sms, TILE_COST_192);
    if (tile_m == 192 || p192.us < plan.us) { plan = p192; bm = 192; }
  }
  int split = plan.split;
  YMP_CHECK_ARG(split == 1 || (a->accumulate && a->out_dtype == YMP_DT_F32), "ymp_gemm: split_k>1 needs accumulate=1 and fp32 output");
  if (split > kb_total) split = kb_total;
  int per = (kb_total + split - 1) / split;
  split = (kb_total + per - 1) / per;  // no empty splits

  GemmKParams kp;
  kp.D = a->D;
  kp.bias = reinterpret_cast<const __nv_bfloat16*>(a->bias);
  kp.residual = a->residual;
  kp.res_f32 = (a->residual_dtype == YMP_DT_F32) ? 1 : 0;
  kp.aux_out = reinterpret_cast<__nv_bfloat16*>(a->aux_out);
  kp.aux_in = reinterpret_cast<const __nv_bfloat16*>(a->aux_in);
  kp.M = a->M; kp.N = a->N; kp.K = a->K;
  kp.ldd = a->ldd; kp.ldr = a->ldr;
  kp.a_mn = a->a_mn_major ? 1 : 0; kp.b_mn = a->b_mn_major ? 1 : 0;
  kp.act = a->act; kp.out_f32 = (a->out_dtype == YMP_DT_F32); kp.accumulate = a->accumulate ? 1 : 0;
  kp.split_k = split; kp.kb_per_split = per;
  kp.alpha = a->alpha;
  // keep the larger operand streaming once from HBM: the smaller one is the re-read (L2-resident) side
  kp.n_fast = ((long)a->M >= (long)a->N) ? 1 : 0;
  kp.res_row_mod = a->res_row_mod; kp.d_row_block = a->d_row_block; kp.d_row_stride = a->d_row_stride;
  kp.im2col_T = a->im2col_P ? a->im2col_T : 0;
  kp.im2col_Wp = a->im2col_P ? a->im2col_W / a->im2col_P : 0;
  kp.im2col_N = a->im2col_P ? (a->im2col_H / a->im2col_P) * kp.im2col_Wp : 0;
  kp.has_drop = (a->drop.rng && a->drop.p > 0.f) ? 1 : 0;
  kp.drop.rng = a->drop.rng; kp.drop.site = a->drop.site; kp.drop.p = a->drop.p;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool partial = g_deterministic && split > 1;
  if (ws_bytes) {
    *ws_bytes = partial ? (int64_t)split * a->M * a->ldd * sizeof(float) : 0;
    return YMP_OK;
  }
  if (partial) {
    YMP_CHECK_ARG(workspace && aligned16(workspace), "ymp_gemm: deterministic split-K needs a 16-byte aligned workspace of "
                  "ymp_gemm_workspace_size bytes (ymp_gemm_ws)");
    YMP_CHECK_ARG(a->d_row_block == 0, "ymp_gemm: deterministic split-K does not take d_row_block");
    kp.D = workspace;
    kp.accumulate = 0;
    const int rc = bm == 192 ? launch_gemm<192, 256, true>(a, kp, st)
                   : bn == 256 ? launch_gemm<128, 256, true>(a, kp, st) : launch_gemm<128, 128, true>(a, kp, st);
    if (rc) return rc;
    return ordered_sum(reinterpret_cast<float*>(a->D), a->ldd, reinterpret_cast<const float*>(workspace), a->ldd,
                       (long)a->M * a->ldd, a->M, a->N, split, st);
  }
  if (bm == 192) return launch_gemm<192, 256>(a, kp, st);
  if (bn == 256) return launch_gemm<128, 256>(a, kp, st);
  return launch_gemm<128, 128>(a, kp, st);
}
}  // namespace ymp

extern "C" int ymp_gemm(const ymp_gemm_args* a, void* stream) { return ymp_gemm_tiled(a, 0, stream); }

extern "C" int ymp_gemm_tiled(const ymp_gemm_args* a, int tile_m, void* stream) { return ymp::gemm_run(a, tile_m, nullptr, stream, nullptr); }

extern "C" int ymp_gemm_ws(const ymp_gemm_args* a, int tile_m, void* workspace, void* stream) {
  return ymp::gemm_run(a, tile_m, workspace, stream, nullptr);
}

extern "C" int64_t ymp_gemm_workspace_size(const ymp_gemm_args* a, int tile_m) {
  int64_t bytes = 0;
  const int rc = ymp::gemm_run(a, tile_m, nullptr, nullptr, &bytes);
  return rc ? rc : bytes;
}
