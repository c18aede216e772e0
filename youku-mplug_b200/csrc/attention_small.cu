// Block-diagonal attention over SHORT dense sequences (length T <= 16): the TimeSformer temporal attention
// (T frames of one patch are T consecutive rows, models/vision_transformer.py:246-248 of the reference).
//
// One WARP owns floor(16 / T) whole sequences (<= 16 rows) of one head and never talks to another warp:
//   forward : cp.async Q,K,V rows -> S = Q K^T (mma.sync m16n8k16, 16x16 scores) -> masked exact softmax in
//             registers -> O = P V -> rows staged in smem -> 16-byte coalesced stores (+ lse)
//   backward: one fused kernel (dQ, dK, dV; no delta workspace, O is not read):
//             P = exp(S - lse), dP = dO V^T, delta = rowsum(P o dP) (== rowsum(dO o O)), dS = P o (dP - delta),
//             dQ = dS K, dV = P^T dO, dK = dS^T Q with the transposed fragments made by movmatrix
// The kernels are HBM-bound (a few hundred bytes of arithmetic per row); the design goal is bytes in flight:
// ~10-13 KB of cp.async per warp, 16-20 resident warps per SM, no block-level barriers.
#include <math_constants.h>

#include "common.h"
#include "ptx.cuh"

namespace ymp {

struct SmallParams {
  const __nv_bfloat16 *q, *k, *v, *dout;
  __nv_bfloat16 *o, *dq, *dk, *dv;
  float* lse;
  int ldq, ldk, ldv, ldo, lddo, lddq, lddk, lddv;
  int hsq, hsk, hsv, hso, hsdo, hsdq, hsdk, hsdv;
  int n_heads, T, P, rows_w, n_tiles;
  long R;
  float scale_log2, scale;
};

namespace {
__device__ __forceinline__ uint32_t sm_movt(uint32_t a) {
  uint32_t d;
  asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(d) : "r"(a));
  return d;
}
__device__ __forceinline__ float sm_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 16 rows x HD columns of one operand -> smem tile [16][PITCH]; rows >= nrows are zero-filled
template <int HD>
__device__ __forceinline__ void load16(uint8_t* tile, const __nv_bfloat16* base, long ld, int nrows, int lane) {
  constexpr int CPR = HD / 8, PITCH = HD * 2 + 16;
#pragma unroll
  for (int j = 0; j < (16 * CPR + 31) / 32; ++j) {
    const int c = lane + 32 * j;
    if (c < 16 * CPR) {
      const int r = c / CPR, cc = c - r * CPR;
      if (r < nrows) cp_async16(tile + r * PITCH + cc * 16, base + (long)r * ld + cc * 8);
      else *reinterpret_cast<uint4*>(tile + r * PITCH + cc * 16) = make_uint4(0, 0, 0, 0);
    }
  }
}
// staged [16][PITCH] rows -> global, 16-byte coalesced
template <int HD>
__device__ __forceinline__ void store16(const uint8_t* tile, __nv_bfloat16* base, long ld, int nrows, int lane) {
  constexpr int CPR = HD / 8, PITCH = HD * 2 + 16;
#pragma unroll
  for (int j = 0; j < (16 * CPR + 31) / 32; ++j) {
    const int c = lane + 32 * j;
    if (c < 16 * CPR) {
      const int r = c / CPR, cc = c - r * CPR;
      if (r < nrows) *reinterpret_cast<uint4*>(base + (long)r * ld + cc * 8) = *reinterpret_cast<const uint4*>(tile + r * PITCH + cc * 16);
    }
  }
}
// accumulator fragments [HD/8][4] (x mul) -> staged bf16 rows
template <int HD>
__device__ __forceinline__ void stage_acc(uint8_t* tile, const float (&acc)[HD / 8][4], float m0, float m1, int g, int t4) {
  constexpr int PITCH = HD * 2 + 16;
#pragma unroll
  for (int nb = 0; nb < HD / 8; ++nb) {
    *reinterpret_cast<uint32_t*>(tile + g * PITCH + nb * 16 + t4 * 4) = pack_bf16(acc[nb][0] * m0, acc[nb][1] * m0);
    *reinterpret_cast<uint32_t*>(tile + (g + 8) * PITCH + nb * 16 + t4 * 4) = pack_bf16(acc[nb][2] * m1, acc[nb][3] * m1);
  }
}
// C[16 x 16] = A[16 x HD] * B[16 x HD]^T, both tiles row-major in smem
template <int HD>
__device__ __forceinline__ void mma_abt(float (&c)[2][4], const uint8_t* A, const uint8_t* B, int lane) {
  constexpr int PITCH = HD * 2 + 16;
#pragma unroll
  for (int kk = 0; kk < HD / 16; ++kk) {
    uint32_t a[4], b[4];
    ldsm_x4(a, smem_u32(A + (lane & 15) * PITCH + kk * 32 + (lane >> 4) * 16));
    ldsm_x4(b, smem_u32(B + ((lane & 7) + (lane >> 4) * 8) * PITCH + kk * 32 + ((lane >> 3) & 1) * 16));
    mma16816(c[0], a, b[0], b[1]);
    mma16816(c[1], a, b[2], b[3]);
  }
}
// C[16 x HD] = A[16 x 16] (register fragments) * B[16 x HD] (smem tile, rows = contraction index)
template <int HD>
__device__ __forceinline__ void mma_ab(float (&c)[HD / 8][4], const uint32_t (&a)[4], const uint8_t* B, int lane) {
  constexpr int PITCH = HD * 2 + 16;
#pragma unroll
  for (int nb = 0; nb < HD / 8; ++nb) c[nb][0] = c[nb][1] = c[nb][2] = c[nb][3] = 0.f;
#pragma unroll
  for (int dbp = 0; dbp < HD / 16; ++dbp) {
    uint32_t b[4];
    ldsm_x4_t(b, smem_u32(B + ((lane & 7) + ((lane >> 3) & 1) * 8) * PITCH + dbp * 32 + (lane >> 4) * 16));
    mma16816(c[2 * dbp], a, b[0], b[1]);
    mma16816(c[2 * dbp + 1], a, b[2], b[3]);
  }
}
}  // namespace

template <int HD>
__global__ void __launch_bounds__(128) attn_small_fwd_kernel(const SmallParams p) {
  constexpr int PITCH = HD * 2 + 16, TILE = 16 * PITCH;
  extern __shared__ __align__(16) uint8_t smem_small[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const int wt = blockIdx.x * 4 + warp, h = blockIdx.y;
  if (wt >= p.n_tiles) return;
  const long r0 = (long)wt * p.rows_w;
  const int nrows = (int)min((long)p.rows_w, p.R - r0);
  uint8_t* Qs = smem_small + warp * 3 * TILE;
  uint8_t* Ks = Qs + TILE;
  uint8_t* Vs = Ks + TILE;
  load16<HD>(Qs, p.q + r0 * p.ldq + h * p.hsq, p.ldq, nrows, lane);
  load16<HD>(Ks, p.k + r0 * p.ldk + h * p.hsk, p.ldk, nrows, lane);
  load16<HD>(Vs, p.v + r0 * p.ldv + h * p.hsv, p.ldv, nrows, lane);
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncwarp();

  float sc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  mma_abt<HD>(sc, Qs, Ks, lane);
  // element e of n-tile nt: row g + 8 (e >> 1), key column 8 nt + 2 t4 + (e & 1)
  const int blk0 = g / p.T, blk1 = (g + 8) / p.T;
  float mx[2] = {-CUDART_INF_F, -CUDART_INF_F};
  bool ok[2][4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int col = nt * 8 + t4 * 2 + (e & 1);
      ok[nt][e] = (col / p.T == ((e >> 1) ? blk1 : blk0)) && col < nrows;
      if (ok[nt][e]) mx[e >> 1] = fmaxf(mx[e >> 1], sc[nt][e]);
    }
  float l[2] = {0.f, 0.f}, ms[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    ms[r] = (mx[r] == -CUDART_INF_F) ? 0.f : mx[r] * p.scale_log2;
  }
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float pv = ok[nt][e] ? sm_ex2(fmaf(sc[nt][e], p.scale_log2, -ms[e >> 1])) : 0.f;
      sc[nt][e] = pv;
      l[e >> 1] += pv;
    }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
  uint32_t pa[4] = {pack_bf16(sc[0][0], sc[0][1]), pack_bf16(sc[0][2], sc[0][3]), pack_bf16(sc[1][0], sc[1][1]), pack_bf16(sc[1][2], sc[1][3])};
  float o_acc[HD / 8][4];
  mma_ab<HD>(o_acc, pa, Vs, lane);
  const float inv0 = l[0] > 0.f ? 1.f / l[0] : 0.f, inv1 = l[1] > 0.f ? 1.f / l[1] : 0.f;
  __syncwarp();  // every lane is done reading Q
  stage_acc<HD>(Qs, o_acc, inv0, inv1, g, t4);
  __syncwarp();
  store16<HD>(Qs, p.o + r0 * p.ldo + h * p.hso, p.ldo, nrows, lane);
  if (p.lse && t4 == 0) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = g + 8 * r;
      if (row < nrows) {
        const long gr = r0 + row;
        const long s = gr / p.P;
        p.lse[((size_t)s * p.n_heads + h) * p.P + (gr - s * p.P)] = mx[r] * p.scale + logf(l[r]);
      }
    }
  }
}

template <int HD>
__global__ void __launch_bounds__(128) attn_small_bwd_kernel(const SmallParams p) {
  constexpr int PITCH = HD * 2 + 16, TILE = 16 * PITCH;
  extern __shared__ __align__(16) uint8_t smem_small[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const int wt = blockIdx.x * 4 + warp, h = blockIdx.y;
  if (wt >= p.n_tiles) return;
  const long r0 = (long)wt * p.rows_w;
  const int nrows = (int)min((long)p.rows_w, p.R - r0);
  uint8_t* Qs = smem_small + warp * 4 * TILE;
  uint8_t* Ks = Qs + TILE;
  uint8_t* Vs = Ks + TILE;
  uint8_t* Ds = Vs + TILE;
  load16<HD>(Qs, p.q + r0 * p.ldq + h * p.hsq, p.ldq, nrows, lane);
  load16<HD>(Ks, p.k + r0 * p.ldk + h * p.hsk, p.ldk, nrows, lane);
  load16<HD>(Vs, p.v + r0 * p.ldv + h * p.hsv, p.ldv, nrows, lane);
  load16<HD>(Ds, p.dout + r0 * p.lddo + h * p.hsdo, p.lddo, nrows, lane);
  float lse2[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = g + 8 * r;
    lse2[r] = 1e30f;  // rows that do not exist: P = 0
    if (row < nrows) {
      const long gr = r0 + row;
      const long s = gr / p.P;
      lse2[r] = p.lse[((size_t)s * p.n_heads + h) * p.P + (gr - s * p.P)] * 1.4426950408889634f;
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncwarp();

  float sc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}}, dp[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  mma_abt<HD>(sc, Qs, Ks, lane);
  mma_abt<HD>(dp, Ds, Vs, lane);
  const int blk0 = g / p.T, blk1 = (g + 8) / p.T;
  float delta[2] = {0.f, 0.f};
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int col = nt * 8 + t4 * 2 + (e & 1);
      const bool ok = (col / p.T == ((e >> 1) ? blk1 : blk0)) && col < nrows;
      const float pv = ok ? sm_ex2(fmaf(sc[nt][e], p.scale_log2, -lse2[e >> 1])) : 0.f;
      sc[nt][e] = pv;
      delta[e >> 1] = fmaf(pv, dp[nt][e], delta[e >> 1]);
    }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    delta[r] += __shfl_xor_sync(0xffffffffu, delta[r], 1);
    delta[r] += __shfl_xor_sync(0xffffffffu, delta[r], 2);
  }
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) dp[nt][e] = sc[nt][e] * (dp[nt][e] - delta[e >> 1]);  // dS (unscaled)
  // A fragments of P, dS and of their transposes
  const uint32_t pa[4] = {pack_bf16(sc[0][0], sc[0][1]), pack_bf16(sc[0][2], sc[0][3]), pack_bf16(sc[1][0], sc[1][1]), pack_bf16(sc[1][2], sc[1][3])};
  const uint32_t da[4] = {pack_bf16(dp[0][0], dp[0][1]), pack_bf16(dp[0][2], dp[0][3]), pack_bf16(dp[1][0], dp[1][1]), pack_bf16(dp[1][2], dp[1][3])};
  const uint32_t pt[4] = {sm_movt(pa[0]), sm_movt(pa[2]), sm_movt(pa[1]), sm_movt(pa[3])};
  const uint32_t dt[4] = {sm_movt(da[0]), sm_movt(da[2]), sm_movt(da[1]), sm_movt(da[3])};

  float acc[HD / 8][4];
  // dQ = dS K (x scale); V is dead from here on and its tile stages the outputs
  mma_ab<HD>(acc, da, Ks, lane);
  __syncwarp();
  stage_acc<HD>(Vs, acc, p.scale, p.scale, g, t4);
  __syncwarp();
  store16<HD>(Vs, p.dq + r0 * p.lddq + h * p.hsdq, p.lddq, nrows, lane);
  // dV = P^T dO
  mma_ab<HD>(acc, pt, Ds, lane);
  __syncwarp();
  stage_acc<HD>(Vs, acc, 1.f, 1.f, g, t4);
  __syncwarp();
  store16<HD>(Vs, p.dv + r0 * p.lddv + h * p.hsdv, p.lddv, nrows, lane);
  // dK = dS^T Q (x scale)
  mma_ab<HD>(acc, dt, Qs, lane);
  __syncwarp();
  stage_acc<HD>(Vs, acc, p.scale, p.scale, g, t4);
  __syncwarp();
  store16<HD>(Vs, p.dk + r0 * p.lddk + h * p.hsdk, p.lddk, nrows, lane);
}

namespace {
bool dense(const ymp_seqmap& m, int s) {
  return m.seq_div <= 1 && m.n_prefix == 0 && m.pos_stride == 1 && m.outer_stride == s;
}
bool small_domain(const ymp_attn_args* a) {
  if (a->mask != YMP_MASK_BLOCK || a->mask_block < 1 || a->mask_block > 16) return false;
  if (!(a->head_dim == 64 || a->head_dim == 80 || a->head_dim == 96 || a->head_dim == 128)) return false;
  if (a->s_q != a->s_kv || a->s_q % a->mask_block) return false;
  if (!dense(a->map_q, a->s_q) || !dense(a->map_kv, a->s_q) || !dense(a->map_o, a->s_q)) return false;
  if (a->ldq % 8 || a->ldk % 8 || a->ldv % 8 || a->ldo % 8) return false;
  if (a->q_head_stride % 8 || a->k_head_stride % 8 || a->v_head_stride % 8 || a->o_head_stride % 8) return false;
  return true;
}
void fill_small(const ymp_attn_args* a, SmallParams& p) {
  p.q = (const __nv_bfloat16*)a->q; p.k = (const __nv_bfloat16*)a->k; p.v = (const __nv_bfloat16*)a->v;
  p.o = (__nv_bfloat16*)a->o; p.lse = a->lse;
  p.ldq = a->ldq; p.ldk = a->ldk; p.ldv = a->ldv; p.ldo = a->ldo;
  p.hsq = a->q_head_stride; p.hsk = a->k_head_stride; p.hsv = a->v_head_stride; p.hso = a->o_head_stride;
  p.n_heads = a->n_heads; p.T = a->mask_block; p.P = a->s_q;
  p.rows_w = (16 / a->mask_block) * a->mask_block;
  p.R = a->total_rows > 0 ? a->total_rows : (long)a->n_seq * a->s_q;
  p.n_tiles = (int)((p.R + p.rows_w - 1) / p.rows_w);
  p.scale = a->scale; p.scale_log2 = a->scale * 1.4426950408889634f;
}
template <int HD>
int launch_small_fwd(const SmallParams& p, cudaStream_t st) {
  const int smem = 4 * 3 * 16 * (HD * 2 + 16);
  static DeviceOnce once;
  if (once.first()) { YMP_CUDA(cudaFuncSetAttribute(attn_small_fwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); }
  attn_small_fwd_kernel<HD><<<dim3((p.n_tiles + 3) / 4, p.n_heads), 128, smem, st>>>(p);
  YMP_LAUNCH_CHECK();
  return YMP_OK;
}
template <int HD>
int launch_small_bwd(const SmallParams& p, cudaStream_t st) {
  const int smem = 4 * 4 * 16 * (HD * 2 + 16);
  static DeviceOnce once;
  if (once.first()) { YMP_CUDA(cudaFuncSetAttribute(attn_small_bwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); }
  attn_small_bwd_kernel<HD><<<dim3((p.n_tiles + 3) / 4, p.n_heads), 128, smem, st>>>(p);
  YMP_LAUNCH_CHECK();
  return YMP_OK;
}
}  // namespace

// YMP_ENOSUP (no error text) when the call is outside this kernel's domain
int attn_small_fwd_try(const ymp_attn_args* a, cudaStream_t st) {
  if (!small_domain(a)) return YMP_ENOSUP;
  SmallParams p = {};
  fill_small(a, p);
  if (p.n_tiles <= 0) return YMP_OK;
  switch (a->head_dim) {
    case 64: return launch_small_fwd<64>(p, st);
    case 80: return launch_small_fwd<80>(p, st);
    case 96: return launch_small_fwd<96>(p, st);
    default: return launch_small_fwd<128>(p, st);
  }
}

int attn_small_bwd_try(const ymp_attn_bwd_args* b, cudaStream_t st) {
  const ymp_attn_args* a = &b->fwd;
  if (!small_domain(a)) return YMP_ENOSUP;
  if (!dense(b->map_do, a->s_q) || !dense(b->map_dq, a->s_q) || !dense(b->map_dkv, a->s_q)) return YMP_ENOSUP;
  if (b->do_head_stride % 8 || b->dq_head_stride % 8 || b->dk_head_stride % 8 || b->dv_head_stride % 8) return YMP_ENOSUP;
  SmallParams p = {};
  fill_small(a, p);
  if (p.n_tiles <= 0) return YMP_OK;
  p.dout = (const __nv_bfloat16*)b->dout; p.dq = (__nv_bfloat16*)b->dq; p.dk = (__nv_bfloat16*)b->dk; p.dv = (__nv_bfloat16*)b->dv;
  p.lddo = b->lddo; p.lddq = b->lddq; p.lddk = b->lddk; p.lddv = b->lddv;
  p.hsdo = b->do_head_stride; p.hsdq = b->dq_head_stride; p.hsdk = b->dk_head_stride; p.hsdv = b->dv_head_stride;
  switch (a->head_dim) {
    case 64: return launch_small_bwd<64>(p, st);
    case 80: return launch_small_bwd<80>(p, st);
    case 96: return launch_small_bwd<96>(p, st);
    default: return launch_small_bwd<128>(p, st);
  }
}

}  // namespace ymp
