// Warp-specialised bf16 GEMM for sm_90a (one 128 x BN output tile per CTA, BN = 128 or 256).
//   warpgroup 0   : TMA producer   (cp.async.bulk.tensor 2D / 5D, SWIZZLE_128B, NSTAGE-deep mbarrier ring)
//   warpgroups 1-2: consumers      (wgmma.mma_async m64 x BN x 16 each, fp32 accumulators in registers), then the
//                   epilogue: accumulators staged through shared memory -> one thread per row and 32 columns ->
//                   bias / GELU / GELU' / dropout / residual -> bf16 | fp32 | atomic fp32
// Operands may be K-major or MN-major (the transpose bits of wgmma), so the same kernel serves forward (x.W^T),
// dgrad (dy.W) and wgrad (dy^T.x, split-K with fp32 atomics).
#include <cuda.h>

#include "common.h"
#include "philox.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace ymp {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 bf16 = 128 B = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int GEMM_THREADS = 3 * 128;
constexpr int A_STAGE_BYTES = BM * BK * 2;

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

template <int BN>
struct GemmCfg {
  static constexpr int NSTAGE = (BN == 256) ? 4 : 6;    // 192 KB operand ring either way
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STG_LD = BN + 4;                 // fp32 staging row (+4: conflict-free row-per-thread reads)
  static_assert(BM * STG_LD * 4 <= NSTAGE * STAGE_BYTES, "epilogue staging reuses the operand ring");
  static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + 256 + 1024;
};

// 16 consecutive bf16 (32 bytes: one sector) <-> 16 floats, as two 128-bit accesses (the widest of sm_90)
__device__ __forceinline__ void load16(const __nv_bfloat16* p, float (&f)[16]) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(p)), b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
  const uint32_t r[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 8; ++i) { f[2 * i] = bf16_lo(r[i]); f[2 * i + 1] = bf16_hi(r[i]); }
}
__device__ __forceinline__ void store16(__nv_bfloat16* p, const float* f) {
  uint32_t r[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) r[i] = pack_bf16(f[2 * i], f[2 * i + 1]);
  reinterpret_cast<uint4*>(p)[0] = make_uint4(r[0], r[1], r[2], r[3]);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(r[4], r[5], r[6], r[7]);
}

// Global operands of one epilogue chunk (32 columns of one row), fetched before the staged accumulators are
// read back so that their latency overlaps the shared-memory reads.
struct EpiPrefetch {
  uint32_t bias[16];  // 32 bf16
  uint32_t aux[16];   // 32 bf16 (aux_in)
  uint32_t res[32];   // 32 fp32 or 32 bf16 (first 16 words)
};
__device__ __forceinline__ void load32_raw(const __nv_bfloat16* p, uint32_t* r) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(p) + j);
    r[4 * j] = a.x; r[4 * j + 1] = a.y; r[4 * j + 2] = a.z; r[4 * j + 3] = a.w;
  }
}
__device__ __forceinline__ void epilogue_prefetch(const GemmKParams& p, int row, int col0, EpiPrefetch& pf) {
  if (row >= p.M || col0 + 32 > p.N) return;
  if (p.bias) load32_raw(p.bias + col0, pf.bias);
  if (p.aux_in) load32_raw(p.aux_in + (size_t)row * p.ldd + col0, pf.aux);
  if (p.residual) {
    const int rrow = p.res_row_mod ? row % p.res_row_mod : row;
    if (p.res_f32) {
      const float* rf = reinterpret_cast<const float*>(p.residual) + (size_t)rrow * p.ldr + col0;
      const float4* rp = reinterpret_cast<const float4*>(rf);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 a = __ldg(rp + j);
        pf.res[4 * j] = __float_as_uint(a.x); pf.res[4 * j + 1] = __float_as_uint(a.y);
        pf.res[4 * j + 2] = __float_as_uint(a.z); pf.res[4 * j + 3] = __float_as_uint(a.w);
      }
    } else {
      load32_raw(reinterpret_cast<const __nv_bfloat16*>(p.residual) + (size_t)rrow * p.ldr + col0, pf.res);
    }
  }
}

// Epilogue for one thread: 32 consecutive columns of one output row.
template <bool DROP>
__device__ __forceinline__ void epilogue_chunk(const GemmKParams& p, const uint32_t (&r)[32],
                                               int row, int col0, const EpiPrefetch& pf, const DropState& ds) {
  if (row >= p.M || col0 >= p.N) return;
  const bool full = (col0 + 32 <= p.N);
  const int drow = p.d_row_block ? (row / p.d_row_block) * p.d_row_stride + row % p.d_row_block : row;
  const int rrow = p.res_row_mod ? row % p.res_row_mod : row;
  float v[32];
  if (p.alpha == 1.0f) {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]);
  } else {
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(r[i]) * p.alpha;
  }

  if (full) {
    if (p.bias) {
#pragma unroll
      for (int i = 0; i < 16; ++i) { v[2 * i] += bf16_lo(pf.bias[i]); v[2 * i + 1] += bf16_hi(pf.bias[i]); }
    }
    const size_t off = (size_t)row * p.ldd + col0;          // aux tensors: plain rows
    const size_t doff = (size_t)drow * p.ldd + col0;        // D: optionally re-blocked rows
    // aux_out: with an activation it receives act'(v) (what the backward epilogue multiplies by),
    // without one the value itself.  aux_in: a plain multiplier.  Switches are warp-uniform.
    if (p.aux_in) {
#pragma unroll
      for (int i = 0; i < 16; ++i) { v[2 * i] *= bf16_lo(pf.aux[i]); v[2 * i + 1] *= bf16_hi(pf.aux[i]); }
    } else if (p.act == YMP_ACT_GELU_ERF) {
      if (p.aux_out) {
        float d[32];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float x8[8], v8[8], d8[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) x8[e] = v[8 * j + e];
          gelu_erf_both_x8(x8, v8, d8);
#pragma unroll
          for (int e = 0; e < 8; ++e) { v[8 * j + e] = v8[e]; d[8 * j + e] = d8[e]; }
        }
        store16(p.aux_out + off, d);
        store16(p.aux_out + off + 16, d + 16);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float x8[8], v8[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) x8[e] = v[8 * j + e];
          gelu_erf_x8(x8, v8);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[8 * j + e] = v8[e];
        }
      }
    } else if (p.act == YMP_ACT_GELU_TANH) {
      if (p.aux_out) {
        float d[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = gelu_tanh_both(v[i], d[i]);
        store16(p.aux_out + off, d);
        store16(p.aux_out + off + 16, d + 16);
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = gelu_tanh(v[i]);
      }
    } else if (p.aux_out) {
      store16(p.aux_out + off, v);
      store16(p.aux_out + off + 16, v + 16);
    }
    if constexpr (DROP) {  // bias-dropout-add: residual + dropout(x + bias)
#pragma unroll
      for (int j = 0; j < 8; ++j) drop4(ds, (uint32_t)row, (uint32_t)(col0 + 4 * j), v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    }
    if (p.residual) {
      if (p.res_f32) {  // fp32 residual stream
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] += __uint_as_float(pf.res[i]);
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) { v[2 * i] += bf16_lo(pf.res[i]); v[2 * i + 1] += bf16_hi(pf.res[i]); }
      }
    }
    if (!p.out_f32) {
      __nv_bfloat16* dp = reinterpret_cast<__nv_bfloat16*>(p.D) + doff;
      store16(dp, v);
      store16(dp + 16, v + 16);
    } else if (!p.accumulate) {
      float* d = reinterpret_cast<float*>(p.D) + doff;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        reinterpret_cast<float4*>(d)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    } else {
      float* d = reinterpret_cast<float*>(p.D) + doff;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d + 4 * j),
                     "f"(v[4 * j]), "f"(v[4 * j + 1]), "f"(v[4 * j + 2]), "f"(v[4 * j + 3])
                     : "memory");
      }
    }
  } else {
    // ragged N tail: scalar, bounds-checked
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = col0 + i;
      if (col < p.N) {
        float x = v[i];
        if (p.bias) x += __bfloat162float(p.bias[col]);
        const size_t off = (size_t)row * p.ldd + col, doff = (size_t)drow * p.ldd + col;
        if (p.aux_in) {
          x *= __bfloat162float(p.aux_in[off]);
        } else if (p.act == YMP_ACT_GELU_ERF) {
          float d; x = gelu_erf_both(x, d);
          if (p.aux_out) p.aux_out[off] = __float2bfloat16(d);
        } else if (p.act == YMP_ACT_GELU_TANH) {
          float d; x = gelu_tanh_both(x, d);
          if (p.aux_out) p.aux_out[off] = __float2bfloat16(d);
        } else if (p.aux_out) {
          p.aux_out[off] = __float2bfloat16(x);
        }
        if constexpr (DROP) {
          const uint4 w = drop_words(ds, (uint32_t)row, (uint32_t)col >> 2);
          const uint32_t wc = (col & 3) == 0 ? w.x : (col & 3) == 1 ? w.y : (col & 3) == 2 ? w.z : w.w;
          x = wc >= ds.thresh ? x * ds.scale : 0.f;
        }
        if (p.residual)
          x += p.res_f32 ? reinterpret_cast<const float*>(p.residual)[(size_t)rrow * p.ldr + col]
                         : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.residual)[(size_t)rrow * p.ldr + col]);
        if (!p.out_f32) reinterpret_cast<__nv_bfloat16*>(p.D)[doff] = __float2bfloat16(x);
        else if (!p.accumulate) reinterpret_cast<float*>(p.D)[doff] = x;
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
constexpr int IM2COL_SUB_BYTES = BM * 32;  // one 128-row x 16-column sub-tile
__device__ __forceinline__ void load_a_im2col(uint8_t* sa, const CUtensorMap* tma, uint64_t* bar, int m0, int kb,
                                              const GemmKParams& p) {
  const int T = p.im2col_T, c = kb >> 2, y0 = (kb & 3) * 4;
  const int pt = m0 / T;  // first patch (global index b*N + n) of the tile
  for (int i = 0; i < BM / T; ++i) {
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

template <int BN, int AMN, int BMN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                       const GemmKParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int NSTAGE = Cfg::NSTAGE;
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
      mbar_init(&empty_bar[i], 2);  // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================================================================== TMA producer
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        mbar_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
        uint8_t* sa = smem_a + stage * A_STAGE_BYTES;
        uint8_t* sb = smem_b + stage * Cfg::B_STAGE_BYTES;
        if (p.im2col_T) {
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
        if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ======================================================================= consumers: rows 64 (wg - 1) .. +63
  const int cw = wg - 1;
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
        const uint64_t da = p.im2col_T ? make_smem_desc(sa + k * IM2COL_SUB_BYTES + cw * 64 * 32, 16, 256, 3)
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
      prev = stage;
      if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
  }

  // ======================================================================= epilogue
  // Every operand byte has been consumed (the ring holds this tile only), so the ring becomes the fp32 staging tile.
  named_sync(1, 256);
  float* stg = reinterpret_cast<float*>(smem);
  {
    const int lt = threadIdx.x & 127, r0 = cw * 64 + (lt >> 5) * 16 + ((lt & 31) >> 2), c0 = 2 * (lt & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(stg + r0 * Cfg::STG_LD + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + (r0 + 8) * Cfg::STG_LD + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  named_sync(1, 256);
  DropState ds;  // only read when has_drop
  if (p.has_drop) ds = drop_state(p.drop);
  const int et = threadIdx.x - 128, lr = et & (BM - 1), row = m_blk * BM + lr;
#pragma unroll 1
  for (int c = et >> 7; c < BN / 32; c += 2) {
    const int col0 = n_blk * BN + c * 32;
    EpiPrefetch pf;
    epilogue_prefetch(p, row, col0, pf);
    uint32_t r[32];
    const float4* sp = reinterpret_cast<const float4*>(stg + lr * Cfg::STG_LD + c * 32);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 v = sp[j];
      r[4 * j] = __float_as_uint(v.x); r[4 * j + 1] = __float_as_uint(v.y);
      r[4 * j + 2] = __float_as_uint(v.z); r[4 * j + 3] = __float_as_uint(v.w);
    }
    if (p.has_drop) epilogue_chunk<true>(p, r, row, col0, pf, ds);
    else epilogue_chunk<false>(p, r, row, col0, pf, ds);
  }
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

template <int BN, int AMN, int BMN>
static int launch_gemm_t(const CUtensorMap& ta, const CUtensorMap& tb, const GemmKParams& kp, int grid, cudaStream_t stream) {
  using Cfg = GemmCfg<BN>;
  static DeviceOnce once;
  if (once.first())
    YMP_CUDA(cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<BN, AMN, BMN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  Cfg::SMEM_BYTES));
  gemm_bf16_wgmma_kernel<BN, AMN, BMN><<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(ta, tb, kp);
  YMP_LAUNCH_CHECK();
  return YMP_OK;
}

template <int BN>
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
    case 0: return launch_gemm_t<BN, 0, 0>(ta, tb, kp, grid, stream);
    case 1: return launch_gemm_t<BN, 0, 1>(ta, tb, kp, grid, stream);
    case 2: return launch_gemm_t<BN, 1, 0>(ta, tb, kp, grid, stream);
    default: return launch_gemm_t<BN, 1, 1>(ta, tb, kp, grid, stream);
  }
}

}  // namespace ymp

extern "C" int ymp_gemm(const ymp_gemm_args* a, void* stream) {
  using namespace ymp;
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
  YMP_CHECK_ARG(!(a->accumulate && (a->aux_out || a->aux_in || a->act || a->residual)),
                "ymp_gemm: accumulate mode supports only alpha and bias-free linear epilogue");
  YMP_CHECK_ARG(a->res_row_mod >= 0 && a->d_row_block >= 0 && (a->d_row_block == 0 || a->d_row_stride >= a->d_row_block),
                "ymp_gemm: bad res_row_mod / d_row_block / d_row_stride");
  YMP_CHECK_ARG(!(a->drop.rng && a->drop.p > 0.f) || (a->drop.p < 1.f && !a->aux_out && !a->accumulate),
                "ymp_gemm: dropout needs 0 < p < 1 and is not combined with aux_out / accumulate");
  YMP_CHECK_ARG(a->tile_n == 0 || a->tile_n == 128 || a->tile_n == 256 || a->tile_n == 512,
                "ymp_gemm: tile_n must be 0 (auto), 128, 256 or 512 (the widest tile: 256 columns on sm_90)");

  const int kb_total = (a->K + BK - 1) / BK;
  const int sms = num_sms();
  int bn = a->tile_n == 512 ? 256 : a->tile_n;
  if (a->im2col_P && bn == 0) bn = (a->N <= 128) ? 128 : 256;
  if (bn == 0) {
    // the 128x256 tile when it fills the machine (or for split-K accumulation); 128x128 when N is narrow or the
    // wide tile would leave SMs idle
    const long t256 = (long)((a->M + BM - 1) / BM) * ((a->N + 255) / 256);
    bn = (a->N <= 128 || (t256 < sms && a->split_k <= 1 && !a->accumulate)) ? 128 : 256;
  }
  int split = a->split_k;
  if (split <= 0) {
    split = 1;
    if (a->accumulate) {
      const long tiles = (long)((a->M + BM - 1) / BM) * ((a->N + bn - 1) / bn);
      // cost model (k-blocks of MMA time): waves x (k-blocks per unit + a fixed pipeline-fill / atomic-epilogue
      // overhead of ~24 k-blocks), one unit per SM at a time
      const long workers = sms;
      long best = -1;
      for (int sp = 1; sp <= 64 && sp * 8 <= kb_total; ++sp) {
        const long waves = (tiles * sp + workers - 1) / workers;
        const long cost = waves * ((kb_total + sp - 1) / sp + 24);
        if (best < 0 || cost < best) { best = cost; split = sp; }
      }
    }
  }
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
  if (bn == 256) return launch_gemm<256>(a, kp, st);
  return launch_gemm<128>(a, kp, st);
}

