// Skinny GEMM for single-token decoding (SURVEY.md 8f N2): y[M, N] = epilogue(x[M, K] . w[N, K]^T) with M <= 64 rows
// (beam width / decode batch; a batched beam search over several clips).  Replaces the GPT-3 layer's linears at the
// KV-cache step of models/modeling_distributed_gpt3.py:868-938,580-595,1348-1350.  With a handful of rows the work is
// one pass over the weight matrix: HBM-bound.  A 128-row tensor-core tile would occupy N/128 CTAs (16 for N = 2048) and
// stream the weights at a fraction of the memory bandwidth; a CUDA-core dot product needs ~2.5 issue slots per weight
// byte-pair (bf16 -> fp32 converts + FMAs for every row) and is issue-bound at a quarter of the bandwidth.  So:
//   * a warp owns 8 output columns and one K slice and feeds tensor-core mma.sync.m16n8k16 (bf16, fp32 accumulate)
//     STRAIGHT FROM GLOBAL MEMORY: lane (g, t) loads 16 bytes (8 consecutive k) of weight row n0+g and of activation
//     row g.  The tensor-core fragment wants k = {2t, 2t+1, 2t+8, 2t+9} per lane - but a dot product does not care in
//     which order k is summed as long as both operands use the same order, so the 8 consecutive elements are simply
//     declared to be those positions of two k-steps (a k permutation inside each 32-element block).  No shared memory,
//     no converts: two loads and two MMAs per 16 weight bytes per lane.  x is the A operand;
//   * M <= 8 (gemm_skinny_kernel): rows 8..15 of the A operand are zero registers;
//     9 <= M <= 64 (gemm_skinny_wide_kernel): the same warp layout, K slices, k permutation and k-block loop, but each
//     weight fragment (the B operand) feeds one MMA per group of 16 activation rows, whose a1/a3 registers carry rows
//     8..15 of the group.  Every output element sees the same MMA chain and the same epilogue as in an M <= 8 call, so
//     row r of an M-row call is bit-identical to the same row computed alone;
//   * the 8 warps of a CTA are `ksplit` K-slices x (8 / ksplit) column tiles (ksplit depends on N and K only); every lane
//     keeps SK_UNROLL = 4 k-blocks (4 x 16 bytes of weights) in flight;
//   * partial sums meet in shared memory and are added in slice order; lane (g, t) of the slice-0 warp owns (row g (+8,
//     +16, ...), columns n0+2t, n0+2t+1) and applies
//       v = acc + bias[n] ; v = gelu(v) (optional) ; v += residual[m, n] (bf16 or fp32) ; store bf16 or fp32
//     (+ an optional second bf16 copy at a device-side row offset: the KV-cache row of the new token; ROW_OFF: one
//     offset per result row, y2_off[m], for sequences at different cache lengths).
// Algorithmic bytes per call: N*K*2 (weights) + M*(K + N)*2..4.  The wide kernel re-reads the activations once per
// 8-column tile (from L2): M*K*2 * N/8 bytes of L2 traffic, 8x the weight bytes at M = 64.
#include "common.h"
#include "ptx.cuh"

namespace ymp {

constexpr int SK_MAXM = 8, SK_TILE_N = 8, SK_WARPS = 8, SK_UNROLL = 4;
constexpr int SK_WIDE_MAXM = 64, SK_WIDE_GROUPS = SK_WIDE_MAXM / 16;

// Both kernels take it as __grid_constant__: the epilogue then reads each field from the parameter bank where it uses
// it.  From a by-value copy the compiler unswitches the k-block loop and the epilogue on the fields (several times the
// code, 114 instead of 84 registers in the wide kernel).
struct SkinnyParams {
  const __nv_bfloat16* x;
  const __nv_bfloat16* w;
  const __nv_bfloat16* bias;
  const void* residual;
  void* y;
  __nv_bfloat16* y2;
  const long long* y2_off;   // device scalar, or [M] per-row offsets (ROW_OFF)
  long long ldy2, y2_stride;
  int M, N, K, ldx, ldw, ldr, ldy;
  int act, res_f32, out_f32, ksplit;
};

// Epilogue of result row m, columns n, n + 1 (the accumulators of one lane): identical for both kernels
template <bool ROW_OFF>
__device__ __forceinline__ void skinny_store(const SkinnyParams& p, int m, int n_base, float acc0, float acc1) {
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int n = n_base + e;
    if (n >= p.N) continue;
    float v = e ? acc1 : acc0;
    if (p.bias) v += __bfloat162float(p.bias[n]);
    if (p.act == YMP_ACT_GELU_TANH) v = gelu_tanh(v);
    else if (p.act == YMP_ACT_GELU_ERF) v = gelu_erf(v);
    if (p.residual)
      v += p.res_f32 ? reinterpret_cast<const float*>(p.residual)[(size_t)m * p.ldr + n]
                     : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.residual)[(size_t)m * p.ldr + n]);
    if (p.out_f32) reinterpret_cast<float*>(p.y)[(size_t)m * p.ldy + n] = v;
    else reinterpret_cast<__nv_bfloat16*>(p.y)[(size_t)m * p.ldy + n] = __float2bfloat16(v);
    if (p.y2) p.y2[(long long)m * p.ldy2 + (ROW_OFF ? p.y2_off[m] : *p.y2_off) * p.y2_stride + n] = __float2bfloat16(v);
  }
}

__device__ __forceinline__ void mma16816_bf16(float (&c)[4], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
  // rows 8..15 of the A operand (a1, a3) are zero: only M <= 8 activation rows exist
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%5}, {%7,%8}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(0u), "r"(a2), "r"(b0), "r"(b1));
}

template <bool ROW_OFF>
__device__ __forceinline__ void gemm_skinny(const SkinnyParams& p) {
  __shared__ float part[SK_WARPS][64];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int ks = p.ksplit, kpart = warp % ks, tile = blockIdx.x * (SK_WARPS / ks) + warp / ks;
  const int n0 = tile * SK_TILE_N;
  const bool live = n0 < p.N;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (live) {
    // 16-byte chunks of the K dimension: chunk c = elements [8c, 8c+8); a k-block is 4 chunks (one per t)
    const int nchunk = p.K >> 3, nblk = (nchunk + 3) >> 2;
    const int b_lo = (int)((long)nblk * kpart / ks), b_hi = (int)((long)nblk * (kpart + 1) / ks);
    const uint4* wr = reinterpret_cast<const uint4*>(p.w + (size_t)min(n0 + g, p.N - 1) * p.ldw);
    const uint4* xr = reinterpret_cast<const uint4*>(p.x + (size_t)min(g, p.M - 1) * p.ldx);
    const bool xrow = g < p.M;
    // two register batches of SK_UNROLL k-blocks: the next batch is requested before the current one is consumed, so a
    // warp always has SK_UNROLL..2*SK_UNROLL x 16 bytes of weights in flight
    uint4 wv[SK_UNROLL], xv[SK_UNROLL];
    auto fetch_w = [&](int b, uint4 (&wd)[SK_UNROLL]) {
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) {
        const int c = (b + u) * 4 + t;
        wd[u] = ((b + u) < b_hi && c < nchunk) ? ld_nc_v4(wr + c) : make_uint4(0, 0, 0, 0);
      }
    };
    auto fetch_x = [&](int b, uint4 (&xd)[SK_UNROLL]) {
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) {
        const int c = (b + u) * 4 + t;
        xd[u] = ((b + u) < b_hi && c < nchunk && xrow) ? __ldg(xr + c) : make_uint4(0, 0, 0, 0);
      }
    };
    fetch_w(b_lo, wv);
    fetch_x(b_lo, xv);
    for (int b = b_lo; b < b_hi; b += SK_UNROLL) {
      uint4 wn[SK_UNROLL], xn[SK_UNROLL];
      fetch_w(b + SK_UNROLL, wn);     // (all-zero past the end of the slice)
      fetch_x(b + SK_UNROLL, xn);
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) {
        mma16816_bf16(acc, xv[u].x, xv[u].y, wv[u].x, wv[u].y);
        mma16816_bf16(acc, xv[u].z, xv[u].w, wv[u].z, wv[u].w);
      }
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) { wv[u] = wn[u]; xv[u] = xn[u]; }
    }
  }
  // acc[0], acc[1] = (row g, columns n0 + 2t, n0 + 2t + 1) summed over this warp's K slice
  if (ks > 1) {
    part[warp][2 * lane] = acc[0];
    part[warp][2 * lane + 1] = acc[1];
    __syncthreads();
    if (kpart == 0)
      for (int j = 1; j < ks; ++j) { acc[0] += part[warp + j][2 * lane]; acc[1] += part[warp + j][2 * lane + 1]; }
  }
  if (live && kpart == 0 && g < p.M) skinny_store<ROW_OFF>(p, g, n0 + 2 * t, acc[0], acc[1]);
}
__global__ void __launch_bounds__(SK_WARPS * 32, 1) gemm_skinny_kernel(const __grid_constant__ SkinnyParams p) {
  gemm_skinny<false>(p);
}
__global__ void __launch_bounds__(SK_WARPS * 32, 1) gemm_skinny_rows_kernel(const __grid_constant__ SkinnyParams p) {
  gemm_skinny<true>(p);
}

// 9 <= M <= 64: gemm_skinny_kernel's grid, warp roles, K slices, weight stream and k-block loop (the same zero-padded
// tail), with one accumulator set per group of 16 rows.  Group j's lane (g, t) holds rows 16j + g (acc[j][0..1])
// and 16j + 8 + g (acc[j][2..3]).  The activation chunks of the k-block being consumed are loaded from global memory
// (L2-resident: every CTA reads them) next to the MMAs; only the weights are double-buffered in registers.
template <bool ROW_OFF>
__device__ __forceinline__ void gemm_skinny_wide(const SkinnyParams& p) {
  __shared__ float part[SK_WARPS][32 * 4 * SK_WIDE_GROUPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int ks = p.ksplit, kpart = warp % ks, tile = blockIdx.x * (SK_WARPS / ks) + warp / ks;
  const int n0 = tile * SK_TILE_N;
  const int groups = (p.M + 15) >> 4;
  const bool live = n0 < p.N;
  float acc[SK_WIDE_GROUPS][4];
#pragma unroll
  for (int j = 0; j < SK_WIDE_GROUPS; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  if (live) {
    const int nchunk = p.K >> 3, nblk = (nchunk + 3) >> 2;
    const int b_lo = (int)((long)nblk * kpart / ks), b_hi = (int)((long)nblk * (kpart + 1) / ks);
    const uint4* wr = reinterpret_cast<const uint4*>(p.w + (size_t)min(n0 + g, p.N - 1) * p.ldw);
    uint4 wv[SK_UNROLL];
    auto fetch_w = [&](int b, uint4 (&wd)[SK_UNROLL]) {
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) {
        const int c = (b + u) * 4 + t;
        wd[u] = ((b + u) < b_hi && c < nchunk) ? ld_nc_v4(wr + c) : make_uint4(0, 0, 0, 0);
      }
    };
    // activation chunk c of row r (zero past the slice, past K and for rows >= M)
    auto fetch_x = [&](int r, int b, int c) {
      return (b < b_hi && c < nchunk && r < p.M) ? __ldg(reinterpret_cast<const uint4*>(p.x + (size_t)r * p.ldx) + c)
                                                 : make_uint4(0, 0, 0, 0);
    };
    fetch_w(b_lo, wv);
    for (int b = b_lo; b < b_hi; b += SK_UNROLL) {
      uint4 wn[SK_UNROLL];
      fetch_w(b + SK_UNROLL, wn);
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) {
        const int c = (b + u) * 4 + t;
#pragma unroll
        for (int j = 0; j < SK_WIDE_GROUPS; ++j) {
          if (j < groups) {
            const uint4 lo = fetch_x(16 * j + g, b + u, c), hi = fetch_x(16 * j + 8 + g, b + u, c);
            const uint32_t a0[4] = {lo.x, hi.x, lo.y, hi.y}, a1[4] = {lo.z, hi.z, lo.w, hi.w};
            mma16816(acc[j], a0, wv[u].x, wv[u].y);
            mma16816(acc[j], a1, wv[u].z, wv[u].w);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < SK_UNROLL; ++u) wv[u] = wn[u];
    }
  }
  if (ks > 1) {
#pragma unroll
    for (int j = 0; j < SK_WIDE_GROUPS; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) part[warp][(j * 4 + e) * 32 + lane] = acc[j][e];
    __syncthreads();
    if (kpart == 0)
      for (int s = 1; s < ks; ++s)
#pragma unroll
        for (int j = 0; j < SK_WIDE_GROUPS; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[j][e] += part[warp + s][(j * 4 + e) * 32 + lane];
  }
  if (live && kpart == 0) {
#pragma unroll
    for (int j = 0; j < SK_WIDE_GROUPS; ++j) {
      if (16 * j + g < p.M) skinny_store<ROW_OFF>(p, 16 * j + g, n0 + 2 * t, acc[j][0], acc[j][1]);
      if (16 * j + 8 + g < p.M) skinny_store<ROW_OFF>(p, 16 * j + 8 + g, n0 + 2 * t, acc[j][2], acc[j][3]);
    }
  }
}
__global__ void __launch_bounds__(SK_WARPS * 32, 1) gemm_skinny_wide_kernel(const __grid_constant__ SkinnyParams p) {
  gemm_skinny_wide<false>(p);
}
__global__ void __launch_bounds__(SK_WARPS * 32, 1) gemm_skinny_wide_rows_kernel(const __grid_constant__ SkinnyParams p) {
  gemm_skinny_wide<true>(p);
}

}  // namespace ymp

using namespace ymp;

// ymp_gemm_skinny (max_m = 8) and ymp_gemm_skinny_wide (max_m = 64): the same arguments, checks and M <= 8 launch.
// row_off (the *_rows entry points): per-row offsets of the second copy in place of a->y2_off_dev.
static int gemm_skinny_call(const ymp_gemm_skinny_args* a, void* stream, int max_m, const int64_t* row_off = nullptr) {
  YMP_CHECK_ARG(a && a->x && a->w && a->y, "ymp_gemm_skinny: null pointer");
  YMP_CHECK_ARG(a->M >= 1 && a->M <= max_m && a->N > 0 && a->K > 0 && a->K % 8 == 0, "ymp_gemm_skinny%s: needs 1 <= M <= %d, K %% 8 == 0 (M=%d K=%d)",
                max_m > SK_MAXM ? "_wide" : "", max_m, a->M, a->K);
  YMP_CHECK_ARG(a->ldx % 8 == 0 && a->ldw % 8 == 0 && a->ldx >= a->K && a->ldw >= a->K && aligned16(a->x) && aligned16(a->w), "ymp_gemm_skinny: x / w rows must be 16-byte aligned");
  YMP_CHECK_ARG(a->act >= 0 && a->act <= 2, "ymp_gemm_skinny: bad act");
  SkinnyParams p;
  p.x = (const __nv_bfloat16*)a->x; p.w = (const __nv_bfloat16*)a->w; p.bias = (const __nv_bfloat16*)a->bias;
  p.residual = a->residual; p.y = a->y;
  if (row_off) {
    YMP_CHECK_ARG(a->y2 && !a->y2_off_dev && a->out_dtype == YMP_DT_BF16,
                  "ymp_gemm_skinny_rows: needs y2, a bf16 result and no y2_off_dev (y2_row_off replaces it)");
  } else {
    YMP_CHECK_ARG(!a->y2 || (a->y2_off_dev && a->out_dtype == YMP_DT_BF16), "ymp_gemm_skinny: y2 needs y2_off_dev and a bf16 result");
  }
  p.y2 = (__nv_bfloat16*)a->y2; p.y2_off = (const long long*)(row_off ? row_off : a->y2_off_dev); p.ldy2 = a->ldy2; p.y2_stride = a->y2_off_stride;
  p.M = a->M; p.N = a->N; p.K = a->K; p.ldx = a->ldx; p.ldw = a->ldw; p.ldr = a->ldr; p.ldy = a->ldy;
  p.act = a->act; p.res_f32 = a->residual_dtype == YMP_DT_F32; p.out_f32 = a->out_dtype == YMP_DT_F32;
  // K slices per CTA (the warps of a CTA that share one 8-column tile): as many as leave >= 4 k-blocks of 32 per slice
  int ks = 1;
  const int ks_max = a->N <= 4096 ? 8 : 4;   // wide outputs get fewer K slices per CTA (more column tiles)
  while (ks < ks_max && a->K / (2 * ks) >= 128) ks *= 2;
  p.ksplit = ks;
  const int tiles = (a->N + SK_TILE_N - 1) / SK_TILE_N, tiles_per_cta = SK_WARPS / ks;
  const int blocks = (tiles + tiles_per_cta - 1) / tiles_per_cta;
  cudaStream_t st = (cudaStream_t)stream;
  if (a->M > SK_MAXM) (row_off ? gemm_skinny_wide_rows_kernel : gemm_skinny_wide_kernel)<<<blocks, SK_WARPS * 32, 0, st>>>(p);
  else (row_off ? gemm_skinny_rows_kernel : gemm_skinny_kernel)<<<blocks, SK_WARPS * 32, 0, st>>>(p);
  YMP_LAUNCH_CHECK();
  return YMP_OK;
}

extern "C" int ymp_gemm_skinny(const ymp_gemm_skinny_args* a, void* stream) { return gemm_skinny_call(a, stream, SK_MAXM); }

extern "C" int ymp_gemm_skinny_wide(const ymp_gemm_skinny_args* a, void* stream) {
  return gemm_skinny_call(a, stream, SK_WIDE_MAXM);
}

extern "C" int ymp_gemm_skinny_rows(const ymp_gemm_skinny_args* a, const int64_t* y2_row_off, void* stream) {
  YMP_CHECK_ARG(y2_row_off, "ymp_gemm_skinny_rows: null y2_row_off");
  return gemm_skinny_call(a, stream, SK_MAXM, y2_row_off);
}

extern "C" int ymp_gemm_skinny_wide_rows(const ymp_gemm_skinny_args* a, const int64_t* y2_row_off, void* stream) {
  YMP_CHECK_ARG(y2_row_off, "ymp_gemm_skinny_wide_rows: null y2_row_off");
  return gemm_skinny_call(a, stream, SK_WIDE_MAXM, y2_row_off);
}
