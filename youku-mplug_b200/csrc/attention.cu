// Fused attention (softmax(scale * Q K^T + mask) V) forward and backward.
//
// Flash-style tiles for any sequence length; the score matrix never touches HBM.  Two kernel families share the
// tiling, masking and softmax: warpgroup MMA (wgmma, head_dim 64 / 80 / 88 / 96: every dense, causal and cross shape
// of the models) and warp-level mma.sync (m16n8k16; head_dim 128, packed block-diagonal masks, the device-side key
// count, a few query rows against a long cache).  head_dim 88 is computed zero-padded to 96 in shared memory.
// Both families hold their accumulators in the same per-warp C-fragment layout, so every step around the MMAs is one
// helper that both call (tile loads, key-tile range, masks, online softmax, dropout, dS, the lse / delta staging and
// the epilogues); each kernel keeps its own MMA issue, shared-memory carving and pipelining.
// Optional dropout of the probabilities (Philox, philox.cuh): the forward drops P after the softmax normaliser, the
// backward regenerates the same bits.  ymp_attn_fwd / ymp_attn_bwd (bottom of the file) dispatch first to
// attention_small.cu (block-diagonal sequences of <= 16 rows: TimeSformer temporal attention) and to the
// single-query decoding kernel, and run everything else here.  ymp_attn_fwd_prefix_table runs the wgmma forward's
// TABLE variant: causal with a key prefix per sequence read from a device table; ymp_attn_fwd_prefix_kv its CACHE
// variant, whose prefix starts with rows of a separate K / V tensor (a prefix's keys computed by an earlier call);
// ymp_attn_fwd_packed its PACKED variant: causal within each of many sequences stored back to back.
//   forward   : CTA = 64 query rows x (seq, head); K/V tiles streamed with cp.async double buffering
//   backward  : two kernels, no atomics, deterministic -
//               dQ   kernel: CTA = 64 query rows, streams K/V   (also emits delta = rowsum(dO*O))
//               dKdV kernel: CTA = 64 key rows,   streams Q/dO
// Sequences are addressed through ymp_seqmap, so Q/K/V are read in place from packed QKV GEMM
// outputs (ViT [3,heads,hd], GPT per-head [q|k|v], TimeSformer per-frame sequences with a shared
// cls row, abstractor cross attention).  Mask modes: none, causal, block-diagonal (packs many
// short TimeSformer temporal sequences into one 64-row tile).
#include <math_constants.h>
#include <stdlib.h>

#include "common.h"
#include "philox.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace ymp {

struct SeqMap {
  int seq_div, n_prefix, prefix_per_seq;
  long outer_stride, inner_stride, pos_stride, prefix_base, prefix_stride;
};
static SeqMap to_map(const ymp_seqmap& m) {
  SeqMap r;
  r.seq_div = m.seq_div > 0 ? m.seq_div : 1;
  r.n_prefix = m.n_prefix; r.prefix_per_seq = m.prefix_per_seq;
  r.outer_stride = m.outer_stride; r.inner_stride = m.inner_stride; r.pos_stride = m.pos_stride;
  r.prefix_base = m.prefix_base; r.prefix_stride = m.prefix_stride;
  return r;
}
// A seqmap resolved for one sequence (done once per CTA: no divisions on the load path).
struct RSeq {
  long base, pos_stride, prefix0;
  int n_prefix;
};
__device__ __forceinline__ RSeq resolve(const SeqMap& m, int s) {
  const int outer = s / m.seq_div, inner = s - outer * m.seq_div;
  RSeq r;
  r.base = (long)outer * m.outer_stride + (long)inner * m.inner_stride;
  r.pos_stride = m.pos_stride;
  r.prefix0 = m.prefix_base + (long)(m.prefix_per_seq ? s : outer) * m.prefix_stride;
  r.n_prefix = m.n_prefix;
  return r;
}
__device__ __forceinline__ long rrow(const RSeq& r, int i) {
  return i < r.n_prefix ? r.prefix0 + i : r.base + (long)(i - r.n_prefix) * r.pos_stride;
}

// One operand matrix of one (sequence, head): element pointer of position i without any division
// or 64-bit multiply chain on the load path.
struct RMat {
  const __nv_bfloat16* base;    // position n_prefix (first regular row), head/column offset applied
  const __nv_bfloat16* prefix;  // position 0 when n_prefix > 0
  long stride;                  // elements between consecutive regular positions
  int ld, n_prefix;
};
__device__ __forceinline__ RMat rmat(const __nv_bfloat16* p, const RSeq& r, int ld, int col_off) {
  RMat m;
  m.base = p + r.base * ld + col_off;
  m.prefix = p + r.prefix0 * ld + col_off;
  m.stride = r.pos_stride * ld;
  m.ld = ld;
  m.n_prefix = r.n_prefix;
  return m;
}
__device__ __forceinline__ const __nv_bfloat16* mrow(const RMat& m, int i) {
  return i < m.n_prefix ? m.prefix + (long)i * m.ld : m.base + (long)(i - m.n_prefix) * m.stride;
}
// A key or value matrix of the prefix-cache variant (ymp_attn_fwd_prefix_kv): positions [0, n0) are rows of the
// prefix cache, the later ones positions 0, 1, ... of m.
struct RMatC {
  RMat m;
  const __nv_bfloat16* cache;  // position 0, head offset applied
  int ldc, n0;
};
__device__ __forceinline__ const __nv_bfloat16* mrow(const RMatC& m, int i) {
  return i < m.n0 ? m.cache + (long)i * m.ldc : mrow(m.m, i - m.n0);
}

constexpr int MASK_NONE = 0, MASK_CAUSAL = 1, MASK_BLOCK = 2;
constexpr float LOG2E = 1.4426950408889634f;  // natural log -> the log2 units of the exp2f softmax

struct AttnKParams {
  const __nv_bfloat16 *q, *k, *v;
  __nv_bfloat16* o;
  float* lse;
  int ldq, ldk, ldv, ldo, hsq, hsk, hsv, hso;
  SeqMap mq, mkv, mo;
  int n_seq, n_heads, s_q, s_kv, mask, mask_block;
  long total_rows;  // >0: dense packed sequences; the last one may be short
  float scale_log2, scale;
  // backward only
  const __nv_bfloat16* dout;
  __nv_bfloat16 *dq, *dk, *dv;
  float* delta;
  int lddo, hsdo, lddq, lddk, lddv, hsdq, hsdk, hsdv;
  SeqMap mdo, mdq, mdkv;
  const int* skv_dev;  // optional device scalar: number of keys that exist (KV-cache decoding under a CUDA graph)
  const int* kv_rows;  // optional device row table (decode kernel only): key j of sequence s is k / v row kv_rows[s * kv_rows_ld + j]
  long kv_rows_ld;
  DropSpec drop;       // dropout of the probabilities (has_drop): row = (seq*heads + head)*s_q + query, column = key
  int has_drop;
  const int* n_prefix; // per-prefix key counts (the wgmma forward's TABLE variant): sequence s has n_prefix[s / mkv.seq_div]
                       // keys before its s_q queries
  const __nv_bfloat16 *kc, *vc;  // prefix cache (CACHE variant): key j < n0 of sequence s is row (s / mkv.seq_div) * n0 + j
  int ldc, hsc, n0;
  const int* starts;   // packed sequences (PACKED variant): sequence s is rows starts[s] .. starts[s + 1] - 1
};

// keep-or-drop of the two adjacent key columns col, col+1 (col even) of `row`: scale or zero in place
__device__ __forceinline__ void drop2(const DropState& ds, uint32_t row, uint32_t col, float& a, float& b) {
  const uint4 w = drop_words(ds, row, col >> 2);
  const uint32_t w0 = (col & 2) ? w.z : w.x, w1 = (col & 2) ? w.w : w.y;
  a = w0 >= ds.thresh ? a * ds.scale : 0.f;
  b = w1 >= ds.thresh ? b * ds.scale : 0.f;
}
// keep-or-drop of the single key column col of `row`: a * scale or zero
__device__ __forceinline__ float drop1(const DropState& ds, uint32_t row, uint32_t col, float a) {
  const uint4 w = drop_words(ds, row, col >> 2);
  const uint32_t c = col & 3, wc = c == 0 ? w.x : c == 1 ? w.y : c == 2 ? w.z : w.w;
  return wc >= ds.thresh ? a * ds.scale : 0.f;
}

// effective lengths of sequence s (short last sequence when total_rows is set)
__device__ __forceinline__ void eff_len(const AttnKParams& p, int s, int& sq, int& skv) {
  sq = p.s_q; skv = p.s_kv;
  if (p.skv_dev) skv = min(skv, *p.skv_dev);
  if (p.total_rows > 0) {
    const long left = p.total_rows - (long)s * p.s_q;
    if (left < sq) sq = (int)left;
    if (left < skv) skv = (int)left;
  }
}
// Warp-uniform test: does this 16-row x 64-col score tile need any masking at all?
__device__ __forceinline__ bool tile_needs_mask(const AttnKParams& p, int row_lo, int col0, int skv) {
  if (col0 + 64 > skv) return true;
  if (p.mask == MASK_CAUSAL) return col0 + 63 > row_lo;
  return p.mask == MASK_BLOCK;
}
// Set masked entries of a C-fragment tile to `fill`.  rows: row_lo + g (+8), cols: col0 + nb*8 + t4*2 (+1)
__device__ __forceinline__ void apply_mask(const AttnKParams& p, float (&sc)[8][4], int row_lo, int col0, int skv,
                                           int g, int t4, float fill) {
  const int r0 = row_lo + g, r1 = r0 + 8;
  int rb0 = 0, rb1 = 0;
  if (p.mask == MASK_BLOCK) { rb0 = r0 / p.mask_block; rb1 = r1 / p.mask_block; }
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = col0 + nb * 8 + t4 * 2 + e;
      bool m0 = col >= skv, m1 = m0;
      if (p.mask == MASK_CAUSAL) { m0 |= col > r0; m1 |= col > r1; }
      else if (p.mask == MASK_BLOCK) { const int cb = col / p.mask_block; m0 |= cb != rb0; m1 |= cb != rb1; }
      if (m0) sc[nb][e] = fill;
      if (m1) sc[nb][2 + e] = fill;
    }
  }
}
// The same rule on a transposed C-fragment tile (rows: keys k_lo + g (+8), cols: queries qi0 + nb*8 + t4*2 (+1)), fill
// -inf.  BLOCK: the caller is served block-diagonal masks (the mma.sync kernels; the wgmma ones never are).
template <bool BLOCK>
__device__ __forceinline__ void apply_mask_t(const AttnKParams& p, float (&st)[8][4], int k_lo, int qi0, int skv, int g,
                                             int t4) {
  bool need = k_lo + 16 > skv;
  if (p.mask == MASK_CAUSAL) need |= k_lo + 15 > qi0;
  if (BLOCK && p.mask == MASK_BLOCK) need = true;
  if (!need) return;
  const int k0 = k_lo + g, k1 = k0 + 8;
  int kb0 = 0, kb1 = 0;
  if (BLOCK && p.mask == MASK_BLOCK) { kb0 = k0 / p.mask_block; kb1 = k1 / p.mask_block; }
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int qc = qi0 + nb * 8 + t4 * 2 + e;
      bool m0 = k0 >= skv, m1 = k1 >= skv;
      if (p.mask == MASK_CAUSAL) { m0 |= k0 > qc; m1 |= k1 > qc; }
      else if (BLOCK && p.mask == MASK_BLOCK) { const int qb = qc / p.mask_block; m0 |= qb != kb0; m1 |= qb != kb1; }
      if (m0) st[nb][e] = -CUDART_INF_F;
      if (m1) st[nb][2 + e] = -CUDART_INF_F;
    }
  }
}

// Key tiles [kv_begin, kv_begin + 64 * ntiles) of the query tile whose rows sit at key positions a_lo .. a_lo + 63
// (sq: the rows that exist, for the block mask); returns ntiles.  BLOCK as for apply_mask_t.
template <bool BLOCK>
__device__ __forceinline__ int key_tiles(const AttnKParams& p, int a_lo, int sq, int skv, int& kv_begin) {
  int kv_end = skv;
  kv_begin = 0;
  if (p.mask == MASK_CAUSAL) kv_end = min(skv, a_lo + 64);
  if (BLOCK && p.mask == MASK_BLOCK) {  // only key blocks that intersect this tile's query blocks
    kv_begin = (a_lo / p.mask_block) * p.mask_block / 64 * 64;
    kv_end = min(skv, ((min(a_lo + 64, sq) - 1) / p.mask_block + 1) * p.mask_block);
  }
  return (kv_end - kv_begin + 63) / 64;
}
// Key columns of tile kv0 that the mma.sync warp of query rows r_lo .. r_lo + 15 needs (warp-uniform): the 16-column
// groups from nb_lo (block mask: only its own diagonal blocks) below column nv
__device__ __forceinline__ void warp_key_span(const AttnKParams& p, int r_lo, int kv0, int skv, int& nv, int& nb_lo) {
  nv = min(64, skv - kv0);
  nb_lo = 0;
  if (p.mask == MASK_CAUSAL) nv = min(nv, r_lo + 16 - kv0);
  if (p.mask == MASK_BLOCK) {
    const int c_lo = (r_lo / p.mask_block) * p.mask_block, c_hi = ((r_lo + 15) / p.mask_block + 1) * p.mask_block;
    nb_lo = max(0, (c_lo - kv0) / 16);
    nv = min(nv, c_hi - kv0);
  }
}

// Online softmax over one 16 x 64 tile of raw scores (the softmax scale is folded into one FFMA per element): sc becomes
// the unnormalised probabilities, the running row maxima m_i and this thread's partial row sums l_i advance, and the
// output accumulator is rescaled to the new maxima.
template <int ND>
__device__ __forceinline__ void softmax_step(const AttnKParams& p, float (&sc)[8][4], float (&m_i)[2], float (&l_i)[2],
                                             float (&o_acc)[ND][4]) {
  float mx[2] = {-CUDART_INF_F, -CUDART_INF_F};
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    mx[0] = fmaxf(mx[0], fmaxf(sc[nb][0], sc[nb][1]));
    mx[1] = fmaxf(mx[1], fmaxf(sc[nb][2], sc[nb][3]));
  }
  float alpha[2], ms[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float mnew = fmaxf(m_i[r], mx[r]);
    ms[r] = (mnew == -CUDART_INF_F) ? 0.f : mnew * p.scale_log2;
    alpha[r] = exp2f(m_i[r] * p.scale_log2 - ms[r]);
    m_i[r] = mnew;
    l_i[r] *= alpha[r];
  }
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float pv = exp2f(fmaf(sc[nb][e], p.scale_log2, -ms[e >> 1]));
      sc[nb][e] = pv;
      l_i[e >> 1] += pv;
    }
  }
#pragma unroll
  for (int i = 0; i < ND; ++i) {
    o_acc[i][0] *= alpha[0]; o_acc[i][1] *= alpha[0];
    o_acc[i][2] *= alpha[1]; o_acc[i][3] *= alpha[1];
  }
}
// Dropout of a 16 x 64 tile of P (forward) or dP (dQ kernel) in place: rows drow0 (+8), key columns kv0 + nb*8 + t4*2
// (+1); the same keep bits and scale in both
__device__ __forceinline__ void drop_tile(const DropState& ds, uint32_t drow0, int kv0, int t4, float (&f)[8][4]) {
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    const uint32_t col = (uint32_t)(kv0 + nb * 8 + t4 * 2);
    drop2(ds, drow0, col, f[nb][0], f[nb][1]);
    drop2(ds, drow0 + 8, col, f[nb][2], f[nb][3]);
  }
}
// dS = P o (dP - delta) in place of the (masked) raw scores sc, with P = exp2(S * scale_log2 - lse) (lse in log2 units)
__device__ __forceinline__ void scores_to_ds(const AttnKParams& p, float (&sc)[8][4], const float (&dp)[8][4],
                                             const float (&lse_r)[2], const float (&del_r)[2]) {
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float pv = exp2f(fmaf(sc[nb][e], p.scale_log2, -lse_r[e >> 1]));
      sc[nb][e] = pv * (dp[nb][e] - del_r[e >> 1]);
    }
  }
}
// The transposed frame of the dK / dV kernels (rows: keys k_lo + g (+8), cols: queries qi0 + nb*8 + t4*2 (+1)):
// st becomes P^T (Z^T = dropout(P)^T under dropout; dV += Z^T dO) and dpt becomes dS^T = P^T o (dZ^T - delta), where
// dZ^T = dropout'(V dO^T).  stat: lse (log2 units; +inf for absent queries, so P = 0) [64] | delta [64] of the query
// tile; qrow0: the dropout row of query qi0.
// QUAD_EXCHANGE: the dropout keep bits of a block come from one Philox call per lane, shared within each quad of lanes;
// otherwise each element makes its own call.  Same bits either way.
template <bool QUAD_EXCHANGE>
__device__ __forceinline__ void probs_t(const AttnKParams& p, const DropState& ds, float (&st)[8][4], float (&dpt)[8][4],
                                        const float* stat, uint32_t qrow0, int k_lo, int lane) {
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int nb = 0; nb < 8; ++nb) {
    // dropout keep bits of the four (query, key) pairs this thread holds, bit e for element e: queries q, q + 1 and keys
    // k0, k1 = k0 + 8.  The four lanes g = 4a .. 4a+3 (same t4) need the same four Philox calls (rows q / q + 1, key
    // groups of k0 / k1), each a different word of them: lane j = g & 3 makes call j and the words are exchanged.
    uint32_t keep = 0xFu;
    if (QUAD_EXCHANGE && p.has_drop) {
      const int j = g & 3;
      const uint32_t qr = qrow0 + (uint32_t)(nb * 8 + t4 * 2 + (j & 1));
      const uint4 w = drop_words(ds, qr, (uint32_t)(k_lo + (g & ~3) + (j >> 1) * 8) >> 2);
      keep = 0;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int comp = (j + r) & 3, c = (j - r) & 3;  // send word comp, receive call c's word j
        const uint32_t v = comp == 0 ? w.x : comp == 1 ? w.y : comp == 2 ? w.z : w.w;
        const uint32_t got = __shfl_sync(0xffffffffu, v, (lane & ~0xC) | (c << 2));
        keep |= (got >= ds.thresh ? 1u : 0u) << c;
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int ql = nb * 8 + t4 * 2 + (e & 1);
      const float pv = exp2f(fmaf(st[nb][e], p.scale_log2, -stat[ql]));
      float dz = dpt[nb][e];
      if (p.has_drop) {
        float kf;
        if constexpr (QUAD_EXCHANGE) {
          kf = (keep >> e) & 1u ? ds.scale : 0.f;
        } else {
          const uint32_t qrow = qrow0 + (uint32_t)ql, key = (uint32_t)(k_lo + g + (e >> 1) * 8);
          kf = drop1(ds, qrow, key, 1.f);
        }
        dz *= kf;
        st[nb][e] = pv * kf;
      } else {
        st[nb][e] = pv;
      }
      dpt[nb][e] = pv * (dz - stat[64 + ql]);
    }
  }
}

// dQ kernels, before the key loop: delta = rowsum(dO o O) of this warp's 16 query rows q_lo .. q_lo + 15 into p.delta
// (for the dK / dV kernel, which runs after this one) and stat[64 + r], their lse in log2 units into stat[r].  Straight
// from global (O is not needed anywhere else): lane -> (row = lane/2, every other 8-column chunk of the head dim =
// lane%2), all 16-byte loads independent.
template <int DIO>
__device__ __forceinline__ void stage_dq_stats(const AttnKParams& p, int s, int h, int q_lo, int sq, const RSeq& mo,
                                               const RSeq& mdo, float* stat) {
  const int lane = threadIdx.x & 31, r = lane >> 1, hf = lane & 1;
  const int qi = q_lo + r;
  float acc = 0.f;
  if (qi < sq) {
    const uint4* orow = reinterpret_cast<const uint4*>(p.o + rrow(mo, qi) * p.ldo + h * p.hso);
    const uint4* drow = reinterpret_cast<const uint4*>(p.dout + rrow(mdo, qi) * p.lddo + h * p.hsdo);
#pragma unroll
    for (int c = hf; c < DIO / 8; c += 2) {
      const uint4 a = __ldg(orow + c), b = __ldg(drow + c);
      acc += bf16_lo(a.x) * bf16_lo(b.x) + bf16_hi(a.x) * bf16_hi(b.x) + bf16_lo(a.y) * bf16_lo(b.y) +
             bf16_hi(a.y) * bf16_hi(b.y) + bf16_lo(a.z) * bf16_lo(b.z) + bf16_hi(a.z) * bf16_hi(b.z) +
             bf16_lo(a.w) * bf16_lo(b.w) + bf16_hi(a.w) * bf16_hi(b.w);
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  if (hf == 0) {
    const size_t li = ((size_t)s * p.n_heads + h) * p.s_q + qi;
    stat[64 + r] = acc;
    stat[r] = (qi < sq) ? p.lse[li] * LOG2E : CUDART_INF_F;
    if (qi < sq) p.delta[li] = acc;
  }
}
// dK / dV kernels, with each Q / dO stage: lse (log2 units; +inf for absent queries) and delta of query rows
// qi0 .. qi0 + 63 into stat[0..63] / stat[64..127].  stat_base: the lse / delta index of query 0 of this (seq, head).
__device__ __forceinline__ void stage_dkdv_stats(const AttnKParams& p, size_t stat_base, int qi0, int sq, float* stat) {
  if (threadIdx.x < 64) {
    const int qi = qi0 + threadIdx.x;
    stat[threadIdx.x] = (qi < sq) ? p.lse[stat_base + qi] * LOG2E : CUDART_INF_F;
    stat[64 + threadIdx.x] = (qi < sq) ? p.delta[stat_base + qi] : 0.f;
  }
}

// Epilogues of a warp's 16 rows (row_lo + g, + 8) from their C fragments; columns DIO..D-1 are never stored.
// Forward: O = o_acc / l (after the quad sums this thread's partial l_i) and lse = m * scale + log(l).
// PACKED: lse is [rows, n_heads], indexed by the output row.
template <int D, int DIO, bool PACKED = false>
__device__ __forceinline__ void store_o_lse(const AttnKParams& p, const float (&o_acc)[D / 8][4], const float (&m_i)[2],
                                            float (&l_i)[2], int row_lo, int sq, int s, int h, const RSeq& mo, int g,
                                            int t4) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_i[r] += __shfl_xor_sync(0xffffffffu, l_i[r], 1);
    l_i[r] += __shfl_xor_sync(0xffffffffu, l_i[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = row_lo + g + r * 8;
    if ((unsigned)qi >= (unsigned)sq) continue;  // (unsigned: the padding rows before query 0 of an offset-causal tile)
    const float inv = l_i[r] > 0.f ? 1.f / l_i[r] : 0.f;
    __nv_bfloat16* orow = p.o + rrow(mo, qi) * p.ldo + h * p.hso;
#pragma unroll
    for (int nb = 0; nb < DIO / 8; ++nb)
      *reinterpret_cast<uint32_t*>(orow + nb * 8 + t4 * 2) = pack_bf16(o_acc[nb][2 * r] * inv, o_acc[nb][2 * r + 1] * inv);
    if (p.lse && t4 == 0) {
      const size_t li = PACKED ? (size_t)rrow(mo, qi) * p.n_heads + h : ((size_t)s * p.n_heads + h) * p.s_q + qi;
      p.lse[li] = m_i[r] * p.scale + logf(l_i[r]);
    }
  }
}
// dQ = scale * dq_acc
template <int D, int DIO>
__device__ __forceinline__ void store_dq(const AttnKParams& p, const float (&dq_acc)[D / 8][4], int row_lo, int sq, int h,
                                         const RSeq& mdq, int g, int t4) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = row_lo + g + r * 8;
    if (qi >= sq) continue;
    __nv_bfloat16* dqrow = p.dq + rrow(mdq, qi) * p.lddq + h * p.hsdq;
#pragma unroll
    for (int nb = 0; nb < DIO / 8; ++nb)
      *reinterpret_cast<uint32_t*>(dqrow + nb * 8 + t4 * 2) = pack_bf16(dq_acc[nb][2 * r] * p.scale, dq_acc[nb][2 * r + 1] * p.scale);
  }
}
// dK = scale * dk_acc, dV = dv_acc (rows are keys)
template <int D, int DIO>
__device__ __forceinline__ void store_dkdv(const AttnKParams& p, const float (&dk_acc)[D / 8][4],
                                           const float (&dv_acc)[D / 8][4], int row_lo, int skv, int h, const RSeq& mdkv,
                                           int g, int t4) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int kvr = row_lo + g + r * 8;
    if (kvr >= skv) continue;
    const long row = rrow(mdkv, kvr);
    __nv_bfloat16* dkrow = p.dk + row * p.lddk + h * p.hsdk;
    __nv_bfloat16* dvrow = p.dv + row * p.lddv + h * p.hsdv;
#pragma unroll
    for (int nb = 0; nb < DIO / 8; ++nb) {
      *reinterpret_cast<uint32_t*>(dkrow + nb * 8 + t4 * 2) = pack_bf16(dk_acc[nb][2 * r] * p.scale, dk_acc[nb][2 * r + 1] * p.scale);
      *reinterpret_cast<uint32_t*>(dvrow + nb * 8 + t4 * 2) = pack_bf16(dv_acc[nb][2 * r], dv_acc[nb][2 * r + 1]);
    }
  }
}

// Shared-memory layout of a [64 x D] bf16 operand tile
enum TileLayout {
  PADDED,       // mma.sync: rows of D + 8 elements (the ldmatrix rows of a 16-byte column fall in different banks)
  SWIZZLE_128B  // wgmma: the K-major layout that TMA writes, 64-column panels of 64 rows x 128 bytes, 16-byte chunk c
                // of row r at chunk c ^ (r & 7)
};
// Asynchronously load a [64 x D] bf16 tile: positions r0..r0+63 of the resolved sequence, zero outside [0, n_valid)
// and in columns DIO..D-1.  rows (the forward's kv_rows table of this sequence, or null): position i is row rows[i] of m.
// M: RMat, or RMatC for the keys and values of the prefix-cache variant.
template <TileLayout L, int D, int DIO, class M>
__device__ __forceinline__ void load_tile(void* dst, const M& m, int r0, int n_valid, const int* rows = nullptr) {
  constexpr int CH = D / 8;
#pragma unroll
  for (int it = 0; it < (64 * CH + 127) / 128; ++it) {
    const int idx = threadIdx.x + it * 128;
    if ((64 * CH) % 128 != 0 && idx >= 64 * CH) break;
    const int r = idx / CH, c = idx - r * CH;
    // (pointer steps as written: one summed byte offset costs the mma.sync backward kernels registers and spills)
    uint8_t* d = L == PADDED ? reinterpret_cast<uint8_t*>(static_cast<__nv_bfloat16*>(dst) + r * (D + 8) + c * 8)
                             : static_cast<uint8_t*>(dst) + (c >> 3) * 8192 + r * 128 + (((c & 7) ^ (r & 7)) << 4);
    // (unsigned: a query tile of an offset-causal call may start before the first query row)
    if ((unsigned)(r0 + r) < (unsigned)n_valid && (DIO == D || c * 8 < DIO))
      cp_async16(d, mrow(m, rows ? __ldg(rows + r0 + r) : r0 + r) + c * 8);
    else *reinterpret_cast<uint4*>(d) = make_uint4(0, 0, 0, 0);
  }
}

// ------------------------------------------------------------------------------ forward
template <int D, int DIO>
__global__ void __launch_bounds__(128) attn_fwd_kernel(const AttnKParams p) {
  constexpr int LDS = D + 8, KS = D / 16, TILE = 64 * LDS;
  extern __shared__ __align__(16) uint8_t smem_attn[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(smem_attn);
  __nv_bfloat16* KVs = Qs + TILE;  // [stage][K|V][TILE]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 64, h = blockIdx.y, s = blockIdx.z;
  const int g = lane >> 2, t4 = lane & 3;
  int sq, skv;
  eff_len(p, s, sq, skv);
  if (q0 >= sq) return;
  // kv_rows (single-query decoding at head_dim 88 / 128): key j is physical row table[j] of k / v
  const int* table = p.kv_rows ? p.kv_rows + s * p.kv_rows_ld : nullptr;
  const RSeq mkv = table ? RSeq{0, 1, 0, 0} : resolve(p.mkv, s), mo = resolve(p.mo, s);
  const RMat Mq = rmat(p.q, resolve(p.mq, s), p.ldq, h * p.hsq);
  const RMat Mk = rmat(p.k, mkv, p.ldk, h * p.hsk), Mv = rmat(p.v, mkv, p.ldv, h * p.hsv);
  int kv_begin;
  const int ntiles = key_tiles<true>(p, q0, sq, skv, kv_begin);

  load_tile<PADDED, D, DIO>(Qs, Mq, q0, sq);
  load_tile<PADDED, D, DIO>(KVs, Mk, kv_begin, skv, table);
  load_tile<PADDED, D, DIO>(KVs + TILE, Mv, kv_begin, skv, table);
  cp_async_commit();

  uint32_t qf[KS][4];
  float o_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f; }
  float m_i[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_i[2] = {0.f, 0.f};
  const bool warp_active = (q0 + warp * 16) < sq;
  DropState ds;  // only read when has_drop
  if (p.has_drop) ds = drop_state(p.drop);
  const uint32_t drow0 = (uint32_t)(((long)s * p.n_heads + h) * p.s_q + q0 + warp * 16 + g);

  for (int t = 0; t < ntiles; ++t) {
    const int kv0 = kv_begin + t * 64;
    __nv_bfloat16* Ks = KVs + (t & 1) * 2 * TILE;
    __nv_bfloat16* Vs = Ks + TILE;
    if (t + 1 < ntiles) {
      __nv_bfloat16* Kn = KVs + ((t + 1) & 1) * 2 * TILE;
      load_tile<PADDED, D, DIO>(Kn, Mk, kv0 + 64, skv, table);
      load_tile<PADDED, D, DIO>(Kn + TILE, Mv, kv0 + 64, skv, table);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (t == 0) {
#pragma unroll
      for (int kk = 0; kk < KS; ++kk)
        ldsm_x4(qf[kk], smem_u32(Qs + (warp * 16 + (lane & 15)) * LDS + kk * 16 + (lane >> 4) * 8));
    }
    if (warp_active) {
      int nv, nb_lo;
      warp_key_span(p, q0 + warp * 16, kv0, skv, nv, nb_lo);
      float sc[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) { sc[i][0] = sc[i][1] = sc[i][2] = sc[i][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
#pragma unroll
        for (int nbp = 0; nbp < 4; ++nbp) {
          if (nbp * 16 < nv && nbp >= nb_lo) {
            uint32_t b[4];
            ldsm_x4(b, smem_u32(Ks + (nbp * 16 + (lane & 7) + (lane >> 4) * 8) * LDS + kk * 16 + ((lane >> 3) & 1) * 8));
            mma16816(sc[2 * nbp], qf[kk], b[0], b[1]);
            mma16816(sc[2 * nbp + 1], qf[kk], b[2], b[3]);
          }
        }
      }
      if (tile_needs_mask(p, q0 + warp * 16, kv0, skv))
        apply_mask(p, sc, q0 + warp * 16, kv0, skv, g, t4, -CUDART_INF_F);
      softmax_step(p, sc, m_i, l_i, o_acc);
      // O = dropout(P) V; the normaliser stays that of the undropped P (softmax, then dropout)
      if (p.has_drop) drop_tile(ds, drow0, kv0, t4, sc);
#pragma unroll
      for (int kk2 = 0; kk2 < 4; ++kk2) {
        if (kk2 * 16 < nv && kk2 >= nb_lo) {
          uint32_t pa[4];
          pa[0] = pack_bf16(sc[2 * kk2][0], sc[2 * kk2][1]);
          pa[1] = pack_bf16(sc[2 * kk2][2], sc[2 * kk2][3]);
          pa[2] = pack_bf16(sc[2 * kk2 + 1][0], sc[2 * kk2 + 1][1]);
          pa[3] = pack_bf16(sc[2 * kk2 + 1][2], sc[2 * kk2 + 1][3]);
#pragma unroll
          for (int dbp = 0; dbp < KS; ++dbp) {
            uint32_t b[4];
            ldsm_x4_t(b, smem_u32(Vs + (kk2 * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + dbp * 16 + (lane >> 4) * 8));
            mma16816(o_acc[2 * dbp], pa, b[0], b[1]);
            mma16816(o_acc[2 * dbp + 1], pa, b[2], b[3]);
          }
        }
      }
    }
    __syncthreads();
  }
  if (!warp_active) return;
  store_o_lse<D, DIO>(p, o_acc, m_i, l_i, q0 + warp * 16, sq, s, h, mo, g, t4);
}

// ------------------------------------------------------------------------------ backward: dQ
// Also writes delta[s,h,i] = sum_d dO[i,d] * O[i,d] for the dKdV kernel (which runs after this one).
template <int D, int DIO>
__global__ void __launch_bounds__(128) attn_bwd_dq_kernel(const AttnKParams p) {
  constexpr int LDS = D + 8, KS = D / 16, TILE = 64 * LDS;
  extern __shared__ __align__(16) uint8_t smem_attn[];
  __nv_bfloat16* Qs = reinterpret_cast<__nv_bfloat16*>(smem_attn);
  __nv_bfloat16* dOs = Qs + TILE;
  __nv_bfloat16* KVs = dOs + TILE;  // [stage][K|V][TILE]
  float* stat = reinterpret_cast<float*>(KVs + 4 * TILE);  // lse(log2)[64], delta[64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 64, h = blockIdx.y, s = blockIdx.z;
  const int g = lane >> 2, t4 = lane & 3;
  int sq, skv;
  eff_len(p, s, sq, skv);
  if (q0 >= sq) return;
  const RSeq mkv = resolve(p.mkv, s), mo = resolve(p.mo, s), mdo = resolve(p.mdo, s), mdq = resolve(p.mdq, s);
  const RMat Mq = rmat(p.q, resolve(p.mq, s), p.ldq, h * p.hsq), Mdo = rmat(p.dout, mdo, p.lddo, h * p.hsdo);
  const RMat Mk = rmat(p.k, mkv, p.ldk, h * p.hsk), Mv = rmat(p.v, mkv, p.ldv, h * p.hsv);
  int kv_begin;
  const int ntiles = key_tiles<true>(p, q0, sq, skv, kv_begin);

  load_tile<PADDED, D, DIO>(Qs, Mq, q0, sq);
  load_tile<PADDED, D, DIO>(dOs, Mdo, q0, sq);
  load_tile<PADDED, D, DIO>(KVs, Mk, kv_begin, skv);
  load_tile<PADDED, D, DIO>(KVs + TILE, Mv, kv_begin, skv);
  cp_async_commit();
  stage_dq_stats<DIO>(p, s, h, q0 + warp * 16, sq, mo, mdo, stat + warp * 16);

  uint32_t qf[KS][4], dof[KS][4];
  float dq_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { dq_acc[i][0] = dq_acc[i][1] = dq_acc[i][2] = dq_acc[i][3] = 0.f; }
  const bool warp_active = (q0 + warp * 16) < sq;
  float lse_r[2], del_r[2];
  DropState ds;  // only read when has_drop
  if (p.has_drop) ds = drop_state(p.drop);
  const uint32_t drow0 = (uint32_t)(((long)s * p.n_heads + h) * p.s_q + q0 + warp * 16 + g);

  for (int t = 0; t < ntiles; ++t) {
    const int kv0 = kv_begin + t * 64;
    __nv_bfloat16* Ks = KVs + (t & 1) * 2 * TILE;
    __nv_bfloat16* Vs = Ks + TILE;
    if (t + 1 < ntiles) {
      __nv_bfloat16* Kn = KVs + ((t + 1) & 1) * 2 * TILE;
      load_tile<PADDED, D, DIO>(Kn, Mk, kv0 + 64, skv);
      load_tile<PADDED, D, DIO>(Kn + TILE, Mv, kv0 + 64, skv);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (t == 0) {
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
        const int off = (warp * 16 + (lane & 15)) * LDS + kk * 16 + (lane >> 4) * 8;
        ldsm_x4(qf[kk], smem_u32(Qs + off));
        ldsm_x4(dof[kk], smem_u32(dOs + off));
      }
      lse_r[0] = stat[warp * 16 + g]; lse_r[1] = stat[warp * 16 + g + 8];
      del_r[0] = stat[64 + warp * 16 + g]; del_r[1] = stat[64 + warp * 16 + g + 8];
    }
    if (warp_active) {
      int nv, nb_lo;
      warp_key_span(p, q0 + warp * 16, kv0, skv, nv, nb_lo);
      float sc[8][4], dp[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        sc[i][0] = sc[i][1] = sc[i][2] = sc[i][3] = 0.f;
        dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
      }
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
#pragma unroll
        for (int nbp = 0; nbp < 4; ++nbp) {
          if (nbp * 16 < nv && nbp >= nb_lo) {
            uint32_t b[4];
            const int off = (nbp * 16 + (lane & 7) + (lane >> 4) * 8) * LDS + kk * 16 + ((lane >> 3) & 1) * 8;
            ldsm_x4(b, smem_u32(Ks + off));
            mma16816(sc[2 * nbp], qf[kk], b[0], b[1]);
            mma16816(sc[2 * nbp + 1], qf[kk], b[2], b[3]);
            ldsm_x4(b, smem_u32(Vs + off));
            mma16816(dp[2 * nbp], dof[kk], b[0], b[1]);
            mma16816(dp[2 * nbp + 1], dof[kk], b[2], b[3]);
          }
        }
      }
      if (tile_needs_mask(p, q0 + warp * 16, kv0, skv))
        apply_mask(p, sc, q0 + warp * 16, kv0, skv, g, t4, -CUDART_INF_F);  // exp2(-inf) = 0
      if (p.has_drop) drop_tile(ds, drow0, kv0, t4, dp);  // dP = dropout'(dO V^T)
      scores_to_ds(p, sc, dp, lse_r, del_r);
#pragma unroll
      for (int kk2 = 0; kk2 < 4; ++kk2) {
        if (kk2 * 16 < nv && kk2 >= nb_lo) {
          uint32_t da[4];
          da[0] = pack_bf16(sc[2 * kk2][0], sc[2 * kk2][1]);
          da[1] = pack_bf16(sc[2 * kk2][2], sc[2 * kk2][3]);
          da[2] = pack_bf16(sc[2 * kk2 + 1][0], sc[2 * kk2 + 1][1]);
          da[3] = pack_bf16(sc[2 * kk2 + 1][2], sc[2 * kk2 + 1][3]);
#pragma unroll
          for (int dbp = 0; dbp < KS; ++dbp) {
            uint32_t b[4];
            ldsm_x4_t(b, smem_u32(Ks + (kk2 * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + dbp * 16 + (lane >> 4) * 8));
            mma16816(dq_acc[2 * dbp], da, b[0], b[1]);
            mma16816(dq_acc[2 * dbp + 1], da, b[2], b[3]);
          }
        }
      }
    }
    __syncthreads();
  }
  if (!warp_active) return;
  store_dq<D, DIO>(p, dq_acc, q0 + warp * 16, sq, h, mdq, g, t4);
}

// ------------------------------------------------------------------------------ backward: dK, dV
template <int D, int DIO>
__global__ void __launch_bounds__(128) attn_bwd_dkdv_kernel(const AttnKParams p) {
  constexpr int LDS = D + 8, KS = D / 16, TILE = 64 * LDS;
  extern __shared__ __align__(16) uint8_t smem_attn[];
  __nv_bfloat16* Ks = reinterpret_cast<__nv_bfloat16*>(smem_attn);
  __nv_bfloat16* Vs = Ks + TILE;
  __nv_bfloat16* QDs = Vs + TILE;  // [stage][Q|dO][TILE]
  float* stat = reinterpret_cast<float*>(QDs + 4 * TILE);  // [stage][lse(log2) 64 | delta 64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kv0 = blockIdx.x * 64, h = blockIdx.y, s = blockIdx.z;
  const int g = lane >> 2, t4 = lane & 3;
  int sq, skv;
  eff_len(p, s, sq, skv);
  if (kv0 >= skv) return;
  const RSeq mkv = resolve(p.mkv, s), mdkv = resolve(p.mdkv, s);
  const RMat Mq = rmat(p.q, resolve(p.mq, s), p.ldq, h * p.hsq), Mdo = rmat(p.dout, resolve(p.mdo, s), p.lddo, h * p.hsdo);
  const RMat Mk = rmat(p.k, mkv, p.ldk, h * p.hsk), Mv = rmat(p.v, mkv, p.ldv, h * p.hsv);
  int q_begin = 0, q_end = sq;
  if (p.mask == MASK_CAUSAL) q_begin = kv0;  // 64-aligned
  if (p.mask == MASK_BLOCK) {
    q_begin = (kv0 / p.mask_block) * p.mask_block / 64 * 64;
    q_end = min(sq, ((min(kv0 + 64, skv) - 1) / p.mask_block + 1) * p.mask_block);
  }
  const int ntiles = (q_end - q_begin + 63) / 64;
  const size_t stat_base = ((size_t)s * p.n_heads + h) * p.s_q;

  auto load_stage = [&](int stage, int qi0) {
    __nv_bfloat16* Qn = QDs + stage * 2 * TILE;
    load_tile<PADDED, D, DIO>(Qn, Mq, qi0, sq);
    load_tile<PADDED, D, DIO>(Qn + TILE, Mdo, qi0, sq);
    stage_dkdv_stats(p, stat_base, qi0, sq, stat + stage * 128);
  };

  load_tile<PADDED, D, DIO>(Ks, Mk, kv0, skv);
  load_tile<PADDED, D, DIO>(Vs, Mv, kv0, skv);
  load_stage(0, q_begin);
  cp_async_commit();

  float dk_acc[D / 8][4], dv_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) {
    dk_acc[i][0] = dk_acc[i][1] = dk_acc[i][2] = dk_acc[i][3] = 0.f;
    dv_acc[i][0] = dv_acc[i][1] = dv_acc[i][2] = dv_acc[i][3] = 0.f;
  }
  const bool warp_active = (kv0 + warp * 16) < skv;
  DropState ds;  // only read when has_drop
  if (p.has_drop) ds = drop_state(p.drop);
  const uint32_t dbase = (uint32_t)stat_base;

  for (int t = 0; t < ntiles; ++t) {
    const int qi0 = q_begin + t * 64;
    __nv_bfloat16* Qs = QDs + (t & 1) * 2 * TILE;
    __nv_bfloat16* dOs = Qs + TILE;
    const float* st = stat + (t & 1) * 128;
    if (t + 1 < ntiles) {
      load_stage((t + 1) & 1, qi0 + 64);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (warp_active) {
      // query columns of this tile this warp needs (warp-uniform)
      int nv = min(64, sq - qi0);
      int nb_lo = 0;  // causal: queries below the first key row of this warp contribute nothing
      if (p.mask == MASK_CAUSAL) nb_lo = max(0, (kv0 + warp * 16 - qi0) / 16);
      if (p.mask == MASK_BLOCK) {  // only the query blocks on this warp's diagonal
        const int k_lo = kv0 + warp * 16;
        const int c_lo = (k_lo / p.mask_block) * p.mask_block, c_hi = ((k_lo + 15) / p.mask_block + 1) * p.mask_block;
        nb_lo = max(0, (c_lo - qi0) / 16);
        nv = min(nv, c_hi - qi0);
      }
      float st_[8][4], dpt[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        st_[i][0] = st_[i][1] = st_[i][2] = st_[i][3] = 0.f;
        dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f;
      }
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
        uint32_t kf[4], vf[4];
        const int aoff = (warp * 16 + (lane & 15)) * LDS + kk * 16 + (lane >> 4) * 8;
        ldsm_x4(kf, smem_u32(Ks + aoff));
        ldsm_x4(vf, smem_u32(Vs + aoff));
#pragma unroll
        for (int nbp = 0; nbp < 4; ++nbp) {
          if (nbp * 16 < nv && nbp >= nb_lo) {
            uint32_t b[4];
            const int off = (nbp * 16 + (lane & 7) + (lane >> 4) * 8) * LDS + kk * 16 + ((lane >> 3) & 1) * 8;
            ldsm_x4(b, smem_u32(Qs + off));
            mma16816(st_[2 * nbp], kf, b[0], b[1]);
            mma16816(st_[2 * nbp + 1], kf, b[2], b[3]);
            ldsm_x4(b, smem_u32(dOs + off));
            mma16816(dpt[2 * nbp], vf, b[0], b[1]);
            mma16816(dpt[2 * nbp + 1], vf, b[2], b[3]);
          }
        }
      }
      apply_mask_t<true>(p, st_, kv0 + warp * 16, qi0, skv, g, t4);
      // This kernel runs at the 255-register limit.  With nvcc 12.9 the quad exchange spills least at head_dim 64 / 80 /
      // 128 and the per-element calls at 88 / 96 (none there; 52 bytes with the exchange).
      probs_t<D != 96>(p, ds, st_, dpt, st, dbase + (uint32_t)qi0, kv0 + warp * 16, lane);
#pragma unroll
      for (int kk2 = 0; kk2 < 4; ++kk2) {
        if (kk2 * 16 < nv && kk2 >= nb_lo) {
          uint32_t pa[4], da[4];
          pa[0] = pack_bf16(st_[2 * kk2][0], st_[2 * kk2][1]);
          pa[1] = pack_bf16(st_[2 * kk2][2], st_[2 * kk2][3]);
          pa[2] = pack_bf16(st_[2 * kk2 + 1][0], st_[2 * kk2 + 1][1]);
          pa[3] = pack_bf16(st_[2 * kk2 + 1][2], st_[2 * kk2 + 1][3]);
          da[0] = pack_bf16(dpt[2 * kk2][0], dpt[2 * kk2][1]);
          da[1] = pack_bf16(dpt[2 * kk2][2], dpt[2 * kk2][3]);
          da[2] = pack_bf16(dpt[2 * kk2 + 1][0], dpt[2 * kk2 + 1][1]);
          da[3] = pack_bf16(dpt[2 * kk2 + 1][2], dpt[2 * kk2 + 1][3]);
#pragma unroll
          for (int dbp = 0; dbp < KS; ++dbp) {
            uint32_t b[4];
            const int off = (kk2 * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS + dbp * 16 + (lane >> 4) * 8;
            ldsm_x4_t(b, smem_u32(dOs + off));
            mma16816(dv_acc[2 * dbp], pa, b[0], b[1]);
            mma16816(dv_acc[2 * dbp + 1], pa, b[2], b[3]);
            ldsm_x4_t(b, smem_u32(Qs + off));
            mma16816(dk_acc[2 * dbp], da, b[0], b[1]);
            mma16816(dk_acc[2 * dbp + 1], da, b[2], b[3]);
          }
        }
      }
    }
    __syncthreads();
  }
  if (!warp_active) return;
  store_dkdv<D, DIO>(p, dk_acc, dv_acc, kv0 + warp * 16, skv, h, mdkv, g, t4);
}

// ------------------------------------------------------------------------------ wgmma kernels (head_dim 64 / 80 / 96)
// The same tiling, masking, softmax and dropout as the mma.sync kernels above, but each CTA is ONE warpgroup whose
// four warps issue warpgroup MMAs together: S / dP tiles are wgmma m64n64k16 with both operands in shared memory, and
// the P.V / dS.K / P^T.dO / dS^T.Q products are wgmma m64nDk16 with the probabilities as the register A operand (the
// m64 accumulator of a warp is exactly the A fragment of the next product) and the shared tile read MN-major.
// Operand tiles are 64 rows x D bf16 in the SWIZZLE_128B layout, filled by cp.async through the seqmaps.
// head_dim 88 is computed as 96 with zero-filled tail columns that are never stored.
template <int D>
struct WgTile {
  static constexpr int BYTES = ((D + 63) / 64) * 8192;
};
// k-step ks (16 head-dim columns) of a tile whose rows are the M / N dimension
__device__ __forceinline__ uint64_t wg_desc_k(uint32_t base, int ks) {
  return make_smem_desc(base + (ks >> 2) * 8192 + (ks & 3) * 32, 16, 1024, 1);
}
// k-step ks (16 rows) of a tile whose rows are the K dimension and whose head-dim columns are N
__device__ __forceinline__ uint64_t wg_desc_mn(uint32_t base, int ks) { return make_smem_desc(base + ks * 2048, 8192, 1024, 1); }

template <int D>
__device__ __forceinline__ void wg_rs(float (&d)[D / 2], const uint32_t (&a)[4], uint64_t db) {
  if constexpr (D == 64) wgmma_rs_m64n64_tb(d, a, db);
  else if constexpr (D == 80) wgmma_rs_m64n80_tb(d, a, db);
  else wgmma_rs_m64n96_tb(d, a, db);
}
// S[64 x 64] = A . B^T over the head dimension (both tiles K-major)
template <int D>
__device__ __forceinline__ void wg_scores(float (&s)[8][4], uint32_t a, uint32_t b) {
  float (&f)[32] = *reinterpret_cast<float(*)[32]>(&s[0][0]);
#pragma unroll
  for (int i = 0; i < 32; ++i) f[i] = 0.f;
  wgmma_fence_acc(f);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk) wgmma_ss_m64n64(f, wg_desc_k(a, kk), wg_desc_k(b, kk));
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_acc(f);
}
// acc[64 x D] += P[64 x 64] . T[64 x D]  (P as bf16 A fragments of its four 16-column k-steps)
template <int D>
__device__ __forceinline__ void wg_pv(float (&acc)[D / 8][4], const float (&pm)[8][4], uint32_t t) {
  float (&f)[D / 2] = *reinterpret_cast<float(*)[D / 2]>(&acc[0][0]);
  uint32_t pa[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    pa[kk][0] = pack_bf16(pm[2 * kk][0], pm[2 * kk][1]);
    pa[kk][1] = pack_bf16(pm[2 * kk][2], pm[2 * kk][3]);
    pa[kk][2] = pack_bf16(pm[2 * kk + 1][0], pm[2 * kk + 1][1]);
    pa[kk][3] = pack_bf16(pm[2 * kk + 1][2], pm[2 * kk + 1][3]);
  }
  wgmma_fence_acc(f);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wg_rs<D>(f, pa[kk], wg_desc_mn(t, kk));
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_acc(f);
}

// The key or value matrix of one (sequence, head) of the forward: m itself, or with CACHE its first n0 positions taken
// from the prefix cache c.
template <bool CACHE>
__device__ __forceinline__ auto with_cache(const RMat& m, const __nv_bfloat16* c, const AttnKParams& p, int s, int h) {
  if constexpr (CACHE) return RMatC{m, c + (long)(s / p.mkv.seq_div) * p.n0 * p.ldc + h * p.hsc, p.ldc, p.n0};
  else return m;
}

// The rows of sequence s: through the seqmap m, or (PACKED) rows r0, r0 + 1, ... of a packed buffer.
template <bool PACKED>
__device__ __forceinline__ RSeq seq_rows(const SeqMap& m, int s, int r0) {
  if constexpr (PACKED) return RSeq{r0, 1, 0, 0};
  else return resolve(m, s);
}

// TABLE: causal with a key prefix per sequence (ymp_attn_fwd_prefix_table): sequence s has qoff = n_prefix[s / seq_div]
// keys before its s_q queries, the first qoff taken from map_kv's prefix rows; s_kv only bounds the grid.
// CACHE (with TABLE, ymp_attn_fwd_prefix_kv): the first n0 of those qoff keys come from the prefix cache, the other
// qoff - n0 from map_kv's prefix rows.  The tile alignment and key range still follow qoff alone.
// PACKED (ymp_attn_fwd_packed; square causal, qoff = 0): sequence s is rows starts[s] .. starts[s + 1] - 1 of q, k, v
// and o, its tiles aligned to its first row; s_q only bounds the grid.
template <int D, int DIO, bool TABLE = false, bool CACHE = false, bool PACKED = false>
__global__ void __launch_bounds__(128) attn_wg_fwd_kernel(const AttnKParams p) {
  constexpr int TB = WgTile<D>::BYTES;
  extern __shared__ uint8_t smem_wg[];
  uint8_t* sm = smem_wg + ((1024u - (smem_u32(smem_wg) & 1023u)) & 1023u);
  uint8_t* Qs = sm;
  uint8_t* KVs = sm + TB;  // [stage][K|V]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, s = blockIdx.z;
  const int g = lane >> 2, t4 = lane & 3;
  // Causal with s_q < s_kv is bottom-right aligned: query i sits at key position i + qoff and sees keys j <= i + qoff.
  // Query tiles are aligned to the key tiles (the first starts qoff % 64 rows before query 0, those rows are padding),
  // so each row meets the same key tiles, masks and arithmetic as the same row of the square causal call over the
  // whole key range: bit-identical O and lse, and no key tile that is fully masked for a row.
  int qoff = p.mask == MASK_CAUSAL ? p.s_kv - p.s_q : 0;
  int q0 = blockIdx.x * 64 - (qoff & 63), a0 = q0 + qoff;  // first query row of the tile and its key position
  if constexpr (TABLE) {
    qoff = __ldg(p.n_prefix + s / p.mkv.seq_div);
    q0 = blockIdx.x * 64 - (qoff & 63);
    a0 = q0 + qoff;
  }
  int sq, skv;
  eff_len(p, s, sq, skv);
  if constexpr (TABLE) skv = qoff + sq;
  int r0 = 0;
  if constexpr (PACKED) {
    r0 = __ldg(p.starts + s);
    sq = skv = __ldg(p.starts + s + 1) - r0;
  }
  if (q0 >= sq) return;  // (TABLE: the grid has a tile for every alignment; the surplus ones end here)
  RSeq mkv = seq_rows<PACKED>(p.mkv, s, r0);
  const RSeq mo = seq_rows<PACKED>(p.mo, s, r0);
  if constexpr (TABLE) mkv.n_prefix = CACHE ? qoff - p.n0 : qoff;
  const RMat Mq = rmat(p.q, seq_rows<PACKED>(p.mq, s, r0), p.ldq, h * p.hsq);
  const auto Mk = with_cache<CACHE>(rmat(p.k, mkv, p.ldk, h * p.hsk), p.kc, p, s, h);
  const auto Mv = with_cache<CACHE>(rmat(p.v, mkv, p.ldv, h * p.hsv), p.vc, p, s, h);
  int kv_begin;
  const int ntiles = key_tiles<false>(p, a0, sq, skv, kv_begin);

  load_tile<SWIZZLE_128B, D, DIO>(Qs, Mq, q0, sq);
  load_tile<SWIZZLE_128B, D, DIO>(KVs, Mk, kv_begin, skv);
  load_tile<SWIZZLE_128B, D, DIO>(KVs + TB, Mv, kv_begin, skv);
  cp_async_commit();

  float o_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f; }
  float m_i[2] = {-CUDART_INF_F, -CUDART_INF_F}, l_i[2] = {0.f, 0.f};
  DropState ds;  // only read when has_drop
  if (p.has_drop) ds = drop_state(p.drop);
  const uint32_t drow0 = (uint32_t)(((long)s * p.n_heads + h) * p.s_q + q0 + warp * 16 + g);

  for (int t = 0; t < ntiles; ++t) {
    const int kv0 = kv_begin + t * 64;
    uint8_t* Ks = KVs + (t & 1) * 2 * TB;
    uint8_t* Vs = Ks + TB;
    if (t + 1 < ntiles) {
      uint8_t* Kn = KVs + ((t + 1) & 1) * 2 * TB;
      load_tile<SWIZZLE_128B, D, DIO>(Kn, Mk, kv0 + 64, skv);
      load_tile<SWIZZLE_128B, D, DIO>(Kn + TB, Mv, kv0 + 64, skv);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async();  // cp.async / zero-fill writes -> visible to the wgmma (async proxy) reads
    __syncthreads();
    float sc[8][4];
    wg_scores<D>(sc, smem_u32(Qs), smem_u32(Ks));
    if (tile_needs_mask(p, a0 + warp * 16, kv0, skv)) apply_mask(p, sc, a0 + warp * 16, kv0, skv, g, t4, -CUDART_INF_F);
    softmax_step(p, sc, m_i, l_i, o_acc);
    // O = dropout(P) V; the normaliser stays that of the undropped P (softmax, then dropout)
    if (p.has_drop) drop_tile(ds, drow0, kv0, t4, sc);
    wg_pv<D>(o_acc, sc, smem_u32(Vs));
    __syncthreads();  // every warpgroup MMA of this stage has retired before it is refilled
  }
  store_o_lse<D, DIO, PACKED>(p, o_acc, m_i, l_i, q0 + warp * 16, sq, s, h, mo, g, t4);
}

// dQ (and delta = rowsum(dO * O) for the dK / dV kernel, which runs after this one)
template <int D, int DIO>
__global__ void __launch_bounds__(128) attn_wg_bwd_dq_kernel(const AttnKParams p) {
  constexpr int TB = WgTile<D>::BYTES;
  extern __shared__ uint8_t smem_wg[];
  uint8_t* sm = smem_wg + ((1024u - (smem_u32(smem_wg) & 1023u)) & 1023u);
  uint8_t* Qs = sm;
  uint8_t* dOs = sm + TB;
  uint8_t* KVs = sm + 2 * TB;  // [stage][K|V]
  float* stat = reinterpret_cast<float*>(sm + 6 * TB);  // lse(log2)[64], delta[64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * 64, h = blockIdx.y, s = blockIdx.z;
  const int g = lane >> 2, t4 = lane & 3;
  int sq, skv;
  eff_len(p, s, sq, skv);
  if (q0 >= sq) return;
  const RSeq mkv = resolve(p.mkv, s), mo = resolve(p.mo, s), mdo = resolve(p.mdo, s), mdq = resolve(p.mdq, s);
  const RMat Mq = rmat(p.q, resolve(p.mq, s), p.ldq, h * p.hsq), Mdo = rmat(p.dout, mdo, p.lddo, h * p.hsdo);
  const RMat Mk = rmat(p.k, mkv, p.ldk, h * p.hsk), Mv = rmat(p.v, mkv, p.ldv, h * p.hsv);
  int kv_begin;
  const int ntiles = key_tiles<false>(p, q0, sq, skv, kv_begin);

  load_tile<SWIZZLE_128B, D, DIO>(Qs, Mq, q0, sq);
  load_tile<SWIZZLE_128B, D, DIO>(dOs, Mdo, q0, sq);
  load_tile<SWIZZLE_128B, D, DIO>(KVs, Mk, kv_begin, skv);
  load_tile<SWIZZLE_128B, D, DIO>(KVs + TB, Mv, kv_begin, skv);
  cp_async_commit();
  stage_dq_stats<DIO>(p, s, h, q0 + warp * 16, sq, mo, mdo, stat + warp * 16);
  float dq_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) { dq_acc[i][0] = dq_acc[i][1] = dq_acc[i][2] = dq_acc[i][3] = 0.f; }
  float lse_r[2], del_r[2];
  DropState ds;  // only read when has_drop
  if (p.has_drop) ds = drop_state(p.drop);
  const uint32_t drow0 = (uint32_t)(((long)s * p.n_heads + h) * p.s_q + q0 + warp * 16 + g);

  for (int t = 0; t < ntiles; ++t) {
    const int kv0 = kv_begin + t * 64;
    uint8_t* Ks = KVs + (t & 1) * 2 * TB;
    uint8_t* Vs = Ks + TB;
    if (t + 1 < ntiles) {
      uint8_t* Kn = KVs + ((t + 1) & 1) * 2 * TB;
      load_tile<SWIZZLE_128B, D, DIO>(Kn, Mk, kv0 + 64, skv);
      load_tile<SWIZZLE_128B, D, DIO>(Kn + TB, Mv, kv0 + 64, skv);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async();
    __syncthreads();
    if (t == 0) {
      lse_r[0] = stat[warp * 16 + g]; lse_r[1] = stat[warp * 16 + g + 8];
      del_r[0] = stat[64 + warp * 16 + g]; del_r[1] = stat[64 + warp * 16 + g + 8];
    }
    float sc[8][4], dp[8][4];
    wg_scores<D>(sc, smem_u32(Qs), smem_u32(Ks));
    wg_scores<D>(dp, smem_u32(dOs), smem_u32(Vs));
    if (tile_needs_mask(p, q0 + warp * 16, kv0, skv)) apply_mask(p, sc, q0 + warp * 16, kv0, skv, g, t4, -CUDART_INF_F);
    if (p.has_drop) drop_tile(ds, drow0, kv0, t4, dp);  // dP = dropout'(dO V^T)
    scores_to_ds(p, sc, dp, lse_r, del_r);
    wg_pv<D>(dq_acc, sc, smem_u32(Ks));
    __syncthreads();
  }
  store_dq<D, DIO>(p, dq_acc, q0 + warp * 16, sq, h, mdq, g, t4);
}

// dK, dV: CTA = 64 key rows, streams Q / dO tiles; everything in the transposed frame (rows = keys, columns = queries)
template <int D, int DIO>
__global__ void __launch_bounds__(128) attn_wg_bwd_dkdv_kernel(const AttnKParams p) {
  constexpr int TB = WgTile<D>::BYTES;
  extern __shared__ uint8_t smem_wg[];
  uint8_t* sm = smem_wg + ((1024u - (smem_u32(smem_wg) & 1023u)) & 1023u);
  uint8_t* Ks = sm;
  uint8_t* Vs = sm + TB;
  uint8_t* QDs = sm + 2 * TB;  // [stage][Q|dO]
  float* stat = reinterpret_cast<float*>(sm + 6 * TB);  // [stage][lse(log2) 64 | delta 64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kv0 = blockIdx.x * 64, h = blockIdx.y, s = blockIdx.z;
  const int g = lane >> 2, t4 = lane & 3;
  int sq, skv;
  eff_len(p, s, sq, skv);
  if (kv0 >= skv) return;
  const RSeq mkv = resolve(p.mkv, s), mdkv = resolve(p.mdkv, s);
  const RMat Mq = rmat(p.q, resolve(p.mq, s), p.ldq, h * p.hsq), Mdo = rmat(p.dout, resolve(p.mdo, s), p.lddo, h * p.hsdo);
  const RMat Mk = rmat(p.k, mkv, p.ldk, h * p.hsk), Mv = rmat(p.v, mkv, p.ldv, h * p.hsv);
  const int q_begin = (p.mask == MASK_CAUSAL) ? kv0 : 0;  // 64-aligned
  const int ntiles = (sq - q_begin + 63) / 64;
  const size_t stat_base = ((size_t)s * p.n_heads + h) * p.s_q;

  auto load_stage = [&](int stage, int qi0) {
    uint8_t* Qn = QDs + stage * 2 * TB;
    load_tile<SWIZZLE_128B, D, DIO>(Qn, Mq, qi0, sq);
    load_tile<SWIZZLE_128B, D, DIO>(Qn + TB, Mdo, qi0, sq);
    stage_dkdv_stats(p, stat_base, qi0, sq, stat + stage * 128);
  };

  load_tile<SWIZZLE_128B, D, DIO>(Ks, Mk, kv0, skv);
  load_tile<SWIZZLE_128B, D, DIO>(Vs, Mv, kv0, skv);
  load_stage(0, q_begin);
  cp_async_commit();

  float dk_acc[D / 8][4], dv_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) {
    dk_acc[i][0] = dk_acc[i][1] = dk_acc[i][2] = dk_acc[i][3] = 0.f;
    dv_acc[i][0] = dv_acc[i][1] = dv_acc[i][2] = dv_acc[i][3] = 0.f;
  }
  DropState ds;  // only read when has_drop
  if (p.has_drop) ds = drop_state(p.drop);
  const uint32_t dbase = (uint32_t)stat_base;

  for (int t = 0; t < ntiles; ++t) {
    const int qi0 = q_begin + t * 64;
    uint8_t* Qs = QDs + (t & 1) * 2 * TB;
    uint8_t* dOs = Qs + TB;
    const float* st = stat + (t & 1) * 128;
    if (t + 1 < ntiles) {
      load_stage((t + 1) & 1, qi0 + 64);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async();
    __syncthreads();
    float st_[8][4], dpt[8][4];
    wg_scores<D>(st_, smem_u32(Ks), smem_u32(Qs));   // S^T = K Q^T
    wg_scores<D>(dpt, smem_u32(Vs), smem_u32(dOs));  // dZ^T = V dO^T
    apply_mask_t<false>(p, st_, kv0 + warp * 16, qi0, skv, g, t4);
    probs_t<true>(p, ds, st_, dpt, st, dbase + (uint32_t)qi0, kv0 + warp * 16, lane);
    wg_pv<D>(dv_acc, st_, smem_u32(dOs));
    wg_pv<D>(dk_acc, dpt, smem_u32(Qs));
    __syncthreads();
  }
  store_dkdv<D, DIO>(p, dk_acc, dv_acc, kv0 + warp * 16, skv, h, mdkv, g, t4);
}

// ------------------------------------------------------------------------------ single-query forward (decoding)
// One query row per (sequence, head) over the KV cache: the step of sample() / beam_search()
// (models/modeling_distributed_gpt3.py:874-938).  Pure streaming: every lane owns whole keys (its D-element K and V rows
// arrive as D/8 independent 16-byte loads), keeps a private un-normalised output row in registers under a warp-uniform
// running maximum, and the 128 private rows meet once at the end through shared memory.  Nothing waits on a tile:
// one round trip to the cache per 128 keys instead of a load / mma.sync / softmax pipeline on a 64-row tile with a
// single live row.  Algorithmic bytes: 2 * s_kv * D * 2 per (sequence, head).
// With a row table (kv_rows) each lane first loads its key's table entry, then that row's K and V: a beam search
// permutes its beams by gathering the small table, and the cache rows are never moved.  The per-key arithmetic and the
// lane <-> key assignment are the same either way, so O and lse are bit-identical to a call on the gathered cache.
// SEQ_LENS (ymp_attn_fwd_seq_lens): skv_dev is a per-sequence array, sequence s attends to its first
// min(s_kv, skv_dev[s]) keys (sequences of one decoding step at different cache lengths).
template <int D, bool SEQ_LENS>
__device__ __forceinline__ void attn_decode(const AttnKParams& p) {
  constexpr int CH = D / 8;
  extern __shared__ __align__(16) uint8_t smem_attn[];
  float (*o_part)[D + 1] = reinterpret_cast<float (*)[D + 1]>(smem_attn);   // [128][D + 1]
  float* l_part = reinterpret_cast<float*>(smem_attn) + 128 * (D + 1);      // [128]
  float* m_part = l_part + 128;                                              // [4]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int h = blockIdx.x, s = blockIdx.y;
  const int* table = p.kv_rows ? p.kv_rows + s * p.kv_rows_ld : nullptr;
  // with a table, mrow(Mk, r) is plain physical row r of k (and of v for Mv)
  const RSeq mkv = table ? RSeq{0, 1, 0, 0} : resolve(p.mkv, s);
  const RMat Mk = rmat(p.k, mkv, p.ldk, h * p.hsk), Mv = rmat(p.v, mkv, p.ldv, h * p.hsv);
  const __nv_bfloat16* qrow = p.q + rrow(resolve(p.mq, s), 0) * p.ldq + h * p.hsq;
  constexpr bool TWO_PHASE = D > 80;   // wide heads: V is requested after K has been consumed (register budget)
  uint4 qv[CH], kv[CH], vv[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) qv[c] = __ldg(reinterpret_cast<const uint4*>(qrow) + c);
  auto row_of = [&](int key) { return table ? __ldg(table + key) : key; };
  auto fetch_k = [&](int row) {
    const uint4* kr = reinterpret_cast<const uint4*>(mrow(Mk, row));
#pragma unroll
    for (int c = 0; c < CH; ++c) kv[c] = __ldg(kr + c);
  };
  auto fetch_v = [&](int row) {
    const uint4* vr = reinterpret_cast<const uint4*>(mrow(Mv, row));
#pragma unroll
    for (int c = 0; c < CH; ++c) vv[c] = __ldg(vr + c);
  };
  // the first 128 keys are requested before the device-side key count is known (rows < s_kv always exist in the cache
  // buffer, and every table entry < s_kv names one; what lies past the count is masked below), so the count's own load
  // is off the critical path
  if (warp * 32 + lane < p.s_kv) {
    const int row = row_of(warp * 32 + lane);
    fetch_k(row);
    if (!TWO_PHASE) fetch_v(row);
  }
  int sq, skv;
  if constexpr (SEQ_LENS) skv = min(p.s_kv, p.skv_dev[s]);
  else eff_len(p, s, sq, skv);
  float o[D];
#pragma unroll
  for (int d = 0; d < D; ++d) o[d] = 0.f;
  float m_run = -CUDART_INF_F, l_run = 0.f;
  for (int k0 = 0; k0 < skv; k0 += 128) {
    const int key = k0 + warp * 32 + lane;
    const bool valid = key < skv;
    if (k0 > 0 && valid) {
      const int row = row_of(key);
      fetch_k(row);
      if (!TWO_PHASE) fetch_v(row);
    }
    float sc = -CUDART_INF_F;
    if (valid) {
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const uint32_t* qp = &qv[c].x; const uint32_t* kp = &kv[c].x;
#pragma unroll
        for (int e = 0; e < 4; ++e) { a0 = fmaf(bf16_lo(qp[e]), bf16_lo(kp[e]), a0); a1 = fmaf(bf16_hi(qp[e]), bf16_hi(kp[e]), a1); }
      }
      sc = (a0 + a1) * p.scale_log2;
    }
    if (TWO_PHASE && valid) fetch_v(row_of(key));   // the table entry again (an L1 hit): no register held across the dot
    const float m_new = fmaxf(m_run, warp_max(sc));   // finite: key k0 + warp*32 is valid whenever this warp has any key
    if (m_new == -CUDART_INF_F) continue;              // (a warp past the end of a short cache)
    const float corr = exp2f(m_run - m_new), pr = valid ? exp2f(sc - m_new) : 0.f;
    l_run = l_run * corr + pr;
    if (valid) {
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const uint32_t* vp = &vv[c].x;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          o[8 * c + 2 * e] = fmaf(pr, bf16_lo(vp[e]), o[8 * c + 2 * e] * corr);
          o[8 * c + 2 * e + 1] = fmaf(pr, bf16_hi(vp[e]), o[8 * c + 2 * e + 1] * corr);
        }
      }
    } else {
#pragma unroll
      for (int d = 0; d < D; ++d) o[d] *= corr;
    }
    m_run = m_new;
  }
#pragma unroll
  for (int d = 0; d < D; ++d) o_part[threadIdx.x][d] = o[d];
  l_part[threadIdx.x] = l_run;
  if (lane == 0) m_part[warp] = m_run;
  __syncthreads();
  const float m_all = fmaxf(fmaxf(m_part[0], m_part[1]), fmaxf(m_part[2], m_part[3]));
  float wgt[4];
#pragma unroll
  for (int w = 0; w < 4; ++w) wgt[w] = m_part[w] == -CUDART_INF_F ? 0.f : exp2f(m_part[w] - m_all);
  float l_all = 0.f;
  for (int r = 0; r < 128; ++r) l_all += l_part[r] * wgt[r >> 5];
  __nv_bfloat16* orow = p.o + rrow(resolve(p.mo, s), 0) * p.ldo + h * p.hso;
  for (int d = threadIdx.x; d < D; d += 128) {
    float acc = 0.f;
    for (int r = 0; r < 128; ++r) acc += o_part[r][d] * wgt[r >> 5];
    orow[d] = __float2bfloat16(acc / l_all);
  }
  if (p.lse && threadIdx.x == 0) p.lse[((long)s * p.n_heads + h) * p.s_q] = (m_all + log2f(l_all)) * 0.6931471805599453f;
}
template <int D>
__global__ void __launch_bounds__(128) attn_decode_kernel(const AttnKParams p) { attn_decode<D, false>(p); }
template <int D>
__global__ void __launch_bounds__(128) attn_decode_lens_kernel(const AttnKParams p) { attn_decode<D, true>(p); }
static int fill_params(const ymp_attn_args* a, AttnKParams& p, const char* who) {
  YMP_CHECK_ARG(a && a->q && a->k && a->v, "%s: null q/k/v", who);
  YMP_CHECK_ARG(a->head_dim == 64 || a->head_dim == 80 || a->head_dim == 88 || a->head_dim == 96 || a->head_dim == 128,
                "%s: head_dim %d not in {64,80,88,96,128}", who, a->head_dim);
  YMP_CHECK_ARG(a->n_seq > 0 && a->n_heads > 0 && a->s_q > 0 && a->s_kv > 0, "%s: bad sizes", who);
  YMP_CHECK_ARG(a->ldq % 8 == 0 && a->ldk % 8 == 0 && a->ldv % 8 == 0 && a->ldo % 8 == 0, "%s: row strides must be multiples of 8", who);
  YMP_CHECK_ARG(a->q_head_stride % 8 == 0 && a->k_head_stride % 8 == 0 && a->v_head_stride % 8 == 0 && a->o_head_stride % 8 == 0, "%s: head strides must be multiples of 8", who);
  YMP_CHECK_ARG(aligned16(a->q) && aligned16(a->k) && aligned16(a->v), "%s: q/k/v must be 16-byte aligned", who);
  YMP_CHECK_ARG(a->mask >= 0 && a->mask <= 2, "%s: mask must be 0 (none), 1 (causal) or 2 (block-diagonal)", who);
  YMP_CHECK_ARG(a->mask == YMP_MASK_NONE || a->s_q == a->s_kv || (a->mask == YMP_MASK_CAUSAL && a->s_q < a->s_kv),
                "%s: block masks need s_q == s_kv, causal needs s_q <= s_kv", who);
  YMP_CHECK_ARG(a->mask != YMP_MASK_BLOCK || a->mask_block > 0, "%s: block mask needs mask_block > 0", who);
  YMP_CHECK_ARG(a->total_rows == 0 || (a->s_q == a->s_kv && a->total_rows > (int64_t)(a->n_seq - 1) * a->s_q),
                "%s: total_rows needs s_q == s_kv and must reach the last sequence", who);
  p.q = (const __nv_bfloat16*)a->q; p.k = (const __nv_bfloat16*)a->k; p.v = (const __nv_bfloat16*)a->v;
  p.o = (__nv_bfloat16*)a->o; p.lse = a->lse;
  p.ldq = a->ldq; p.ldk = a->ldk; p.ldv = a->ldv; p.ldo = a->ldo;
  p.hsq = a->q_head_stride; p.hsk = a->k_head_stride; p.hsv = a->v_head_stride; p.hso = a->o_head_stride;
  p.mq = to_map(a->map_q); p.mkv = to_map(a->map_kv); p.mo = to_map(a->map_o);
  p.n_seq = a->n_seq; p.n_heads = a->n_heads; p.s_q = a->s_q; p.s_kv = a->s_kv;
  p.mask = a->mask; p.mask_block = a->mask_block > 0 ? a->mask_block : 1; p.total_rows = a->total_rows;
  p.scale = a->scale; p.scale_log2 = a->scale * LOG2E;
  p.skv_dev = a->s_kv_dev;
  p.kv_rows = a->kv_rows; p.kv_rows_ld = a->kv_rows_ld;
  p.has_drop = (a->drop.rng && a->drop.p > 0.f) ? 1 : 0;
  p.drop.rng = (const uint64_t*)a->drop.rng; p.drop.site = a->drop.site; p.drop.p = a->drop.p;
  return YMP_OK;
}

// The <D, DIO> instantiation that serves a head_dim: 88 is computed as 96 with zero-filled tail columns.
template <int D_, int DIO_ = D_>
struct HeadDim {
  static constexpr int D = D_, DIO = DIO_;
};
// launch(HeadDim<D, DIO>{}) for a head_dim that fill_params accepted.  WITH_128: the family has head_dim-128 kernels
// (only the mma.sync one; the routing never sends head_dim 128 to the others).
template <bool WITH_128, class F>
static int for_head_dim(int head_dim, F&& launch) {
  switch (head_dim) {
    case 64: return launch(HeadDim<64>{});
    case 80: return launch(HeadDim<80>{});
    case 88: return launch(HeadDim<96, 88>{});
    case 96: return launch(HeadDim<96>{});
  }
  if constexpr (WITH_128) return launch(HeadDim<128>{});
  else return set_error(YMP_EINVAL, "attention: no kernel of this family for head_dim %d", head_dim);
}
// One launch of 128 threads with `smem` bytes of dynamic shared memory (opted in once per device and kernel).
template <void (*K)(AttnKParams)>
static int launch_attn(dim3 grid, int smem, cudaStream_t st, const AttnKParams& p) {
  static DeviceOnce once;
  if (once.first()) { YMP_CUDA(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); }
  K<<<grid, 128, smem, st>>>(p);
  YMP_LAUNCH_CHECK();
  return YMP_OK;
}

template <bool SEQ_LENS = false>
static int launch_decode(const AttnKParams& p, int head_dim, cudaStream_t st) {
  return for_head_dim<false>(head_dim, [&](auto hd) {
    constexpr int D = decltype(hd)::D;
    constexpr auto kernel = SEQ_LENS ? attn_decode_lens_kernel<D> : attn_decode_kernel<D>;
    return launch_attn<kernel>(dim3(p.n_heads, p.n_seq), (128 * (D + 1) + 128 + 4) * 4, st, p);
  });
}
static int launch_wg_fwd(const AttnKParams& p, int head_dim, cudaStream_t st) {
  const int lead = p.mask == MASK_CAUSAL ? (p.s_kv - p.s_q) & 63 : 0;  // padding rows before query 0 (offset causal)
  const dim3 grid((p.s_q + lead + 63) / 64, p.n_heads, p.n_seq);
  return for_head_dim<false>(head_dim, [&](auto hd) {
    using H = decltype(hd);
    return launch_attn<attn_wg_fwd_kernel<H::D, H::DIO>>(grid, 5 * WgTile<H::D>::BYTES + 1024, st, p);
  });
}
// The per-sequence prefix is only known on the device, so the grid has (s_q + 63 + 63) / 64 query tiles: enough for
// any lead of 0 .. 63 padding rows.
template <bool CACHE>
static int launch_wg_fwd_table(const AttnKParams& p, int head_dim, cudaStream_t st) {
  const dim3 grid((p.s_q + 126) / 64, p.n_heads, p.n_seq);
  return for_head_dim<false>(head_dim, [&](auto hd) {
    using H = decltype(hd);
    return launch_attn<attn_wg_fwd_kernel<H::D, H::DIO, true, CACHE>>(grid, 5 * WgTile<H::D>::BYTES + 1024, st, p);
  });
}
// Packed sequences: one query tile per 64 rows of the longest one (p.s_q = max_len); a sequence's surplus tiles end at
// once.
static int launch_wg_fwd_packed(const AttnKParams& p, int head_dim, cudaStream_t st) {
  const dim3 grid((p.s_q + 63) / 64, p.n_heads, p.n_seq);
  return for_head_dim<false>(head_dim, [&](auto hd) {
    using H = decltype(hd);
    return launch_attn<attn_wg_fwd_kernel<H::D, H::DIO, false, false, true>>(grid, 5 * WgTile<H::D>::BYTES + 1024, st, p);
  });
}
static int launch_wg_bwd(const AttnKParams& p, int head_dim, cudaStream_t st) {
  return for_head_dim<false>(head_dim, [&](auto hd) {
    using H = decltype(hd);
    const int smem = 6 * WgTile<H::D>::BYTES + 1024 + 1024;
    const int rc = launch_attn<attn_wg_bwd_dq_kernel<H::D, H::DIO>>(dim3((p.s_q + 63) / 64, p.n_heads, p.n_seq), smem, st, p);
    if (rc) return rc;
    return launch_attn<attn_wg_bwd_dkdv_kernel<H::D, H::DIO>>(dim3((p.s_kv + 63) / 64, p.n_heads, p.n_seq), smem, st, p);
  });
}
static int launch_fwd(const AttnKParams& p, int head_dim, cudaStream_t st) {
  return for_head_dim<true>(head_dim, [&](auto hd) {
    using H = decltype(hd);
    return launch_attn<attn_fwd_kernel<H::D, H::DIO>>(dim3((p.s_q + 63) / 64, p.n_heads, p.n_seq), 5 * 64 * (H::D + 8) * 2, st, p);
  });
}
static int launch_bwd(const AttnKParams& p, int head_dim, cudaStream_t st) {
  return for_head_dim<true>(head_dim, [&](auto hd) {
    using H = decltype(hd);
    const int smem = 6 * 64 * (H::D + 8) * 2 + 1024;
    const int rc = launch_attn<attn_bwd_dq_kernel<H::D, H::DIO>>(dim3((p.s_q + 63) / 64, p.n_heads, p.n_seq), smem, st, p);
    if (rc) return rc;
    return launch_attn<attn_bwd_dkdv_kernel<H::D, H::DIO>>(dim3((p.s_kv + 63) / 64, p.n_heads, p.n_seq), smem, st, p);
  });
}

}  // namespace ymp

namespace ymp {
int attn_small_fwd_try(const ymp_attn_args* a, cudaStream_t st);
int attn_small_bwd_try(const ymp_attn_bwd_args* b, cudaStream_t st);
}

static thread_local int g_attn_path = -1;
extern "C" int ymp_attn_last_path(void) { return g_attn_path; }

extern "C" int ymp_attn_fwd(const ymp_attn_args* a, void* stream) {
  using namespace ymp;
  AttnKParams p = {};
  int rc = fill_params(a, p, "ymp_attn_fwd");
  if (rc) return rc;
  YMP_CHECK_ARG(a->o && aligned16(a->o), "ymp_attn_fwd: bad o");
  cudaStream_t st = (cudaStream_t)stream;
  const bool dropped = p.has_drop;
  YMP_CHECK_ARG(!dropped || a->drop.p < 1.f, "ymp_attn_fwd: dropout p must be < 1");
  if (a->kv_rows) {   // the row table is read by the decode kernel (head_dim 64 / 80 / 96) and the mma.sync tiles (88 / 128)
    YMP_CHECK_ARG(a->s_q == 1 && a->mask == YMP_MASK_NONE && !dropped && a->total_rows == 0,
                  "ymp_attn_fwd: kv_rows needs s_q == 1, mask none, no dropout and no total_rows");
    YMP_CHECK_ARG(a->kv_rows_ld >= a->s_kv, "ymp_attn_fwd: kv_rows_ld must be >= s_kv");
  }
  if (a->mask == YMP_MASK_CAUSAL && a->s_q < a->s_kv) {
    // offset causal (a block of queries at the end of a longer key range): always the wgmma tiles, whatever s_q, so
    // that every row is bit-identical to the same row of the square causal call over the whole range
    YMP_CHECK_ARG(a->head_dim != 128, "ymp_attn_fwd: causal with s_q < s_kv needs head_dim 64, 80, 88 or 96");
    YMP_CHECK_ARG(!dropped, "ymp_attn_fwd: causal with s_q < s_kv takes no dropout");
    YMP_CHECK_ARG(!a->s_kv_dev, "ymp_attn_fwd: causal with s_q < s_kv takes no s_kv_dev");
    g_attn_path = YMP_ATTN_PATH_WGMMA;
    return launch_wg_fwd(p, a->head_dim, st);
  }
  if (a->s_q == 1 && a->mask == YMP_MASK_NONE && a->total_rows == 0 && !dropped && a->head_dim != 88 && a->head_dim != 128) {
    g_attn_path = YMP_ATTN_PATH_DECODE;   // one query row per sequence: the streaming kernel (also follows s_kv_dev)
    return launch_decode(p, a->head_dim, st);
  }
  const bool dev_len = a->s_kv_dev != nullptr;  // key count read on the device: the mma.sync kernels bound their KV loop by it
  YMP_CHECK_ARG(!dev_len || (!dropped && a->mask == YMP_MASK_NONE && a->total_rows == 0 && a->head_dim != 88),
                "ymp_attn_fwd: s_kv_dev needs mask none, no dropout, no total_rows, head_dim in {64,80,96,128}");
  if (!dropped && !dev_len && !a->kv_rows) {
    rc = attn_small_fwd_try(a, st);  // short dense block-diagonal sequences (attention_small.cu)
    if (rc != YMP_ENOSUP) { g_attn_path = YMP_ATTN_PATH_SMALL; return rc; }
  }
  // warpgroup-MMA tiles for head_dim <= 96; the mma.sync tiles for head_dim 128, the packed block-diagonal mask (they
  // skip the masked chunks warp by warp), the device-side key count, a row table and a few query rows against a long cache
  if (a->head_dim != 128 && a->mask != YMP_MASK_BLOCK && !dev_len && !a->kv_rows && !(a->s_q < 16 && a->s_kv > 256)) {
    g_attn_path = YMP_ATTN_PATH_WGMMA;
    return launch_wg_fwd(p, a->head_dim, st);
  }
  g_attn_path = YMP_ATTN_PATH_MMA_SYNC;
  return launch_fwd(p, a->head_dim, st);
}

extern "C" int ymp_attn_fwd_seq_lens(const ymp_attn_args* a, const int32_t* kv_lens, void* stream) {
  using namespace ymp;
  AttnKParams p = {};
  int rc = fill_params(a, p, "ymp_attn_fwd_seq_lens");
  if (rc) return rc;
  YMP_CHECK_ARG(kv_lens != nullptr, "ymp_attn_fwd_seq_lens: null kv_lens");
  YMP_CHECK_ARG(a->o && aligned16(a->o), "ymp_attn_fwd_seq_lens: bad o");
  YMP_CHECK_ARG(a->s_q == 1 && a->mask == YMP_MASK_NONE && !p.has_drop && a->total_rows == 0,
                "ymp_attn_fwd_seq_lens: needs s_q == 1, mask none, no dropout and no total_rows");
  YMP_CHECK_ARG(a->head_dim != 88 && a->head_dim != 128, "ymp_attn_fwd_seq_lens: needs head_dim 64, 80 or 96");
  YMP_CHECK_ARG(!a->s_kv_dev, "ymp_attn_fwd_seq_lens: takes no s_kv_dev (kv_lens replaces it)");
  YMP_CHECK_ARG(!a->kv_rows || a->kv_rows_ld >= a->s_kv, "ymp_attn_fwd_seq_lens: kv_rows_ld must be >= s_kv");
  p.skv_dev = kv_lens;
  g_attn_path = YMP_ATTN_PATH_DECODE;
  return launch_decode<true>(p, a->head_dim, (cudaStream_t)stream);
}

// The checks and parameters that ymp_attn_fwd_prefix_table and ymp_attn_fwd_prefix_kv share.
static int fill_table_params(const ymp_attn_prefix_table_args* t, ymp::AttnKParams& p, const char* who) {
  using namespace ymp;
  YMP_CHECK_ARG(t->n_prefix != nullptr, "%s: null n_prefix table", who);
  const ymp_attn_args* a = &t->attn;
  int rc = fill_params(a, p, who);
  if (rc) return rc;
  YMP_CHECK_ARG(a->o && aligned16(a->o), "%s: bad o", who);
  YMP_CHECK_ARG(a->mask == YMP_MASK_CAUSAL, "%s: the mask must be causal", who);
  YMP_CHECK_ARG(a->head_dim != 128, "%s: needs head_dim 64, 80, 88 or 96", who);
  YMP_CHECK_ARG(!p.has_drop, "%s: takes no dropout", who);
  YMP_CHECK_ARG(a->total_rows == 0 && !a->s_kv_dev && !a->kv_rows, "%s: takes no total_rows, s_kv_dev or kv_rows", who);
  p.n_prefix = t->n_prefix;
  return YMP_OK;
}

extern "C" int ymp_attn_fwd_prefix_table(const ymp_attn_prefix_table_args* t, void* stream) {
  using namespace ymp;
  YMP_CHECK_ARG(t != nullptr, "ymp_attn_fwd_prefix_table: null args");
  AttnKParams p = {};
  const int rc = fill_table_params(t, p, "ymp_attn_fwd_prefix_table");
  if (rc) return rc;
  g_attn_path = YMP_ATTN_PATH_WGMMA;
  return launch_wg_fwd_table<false>(p, t->attn.head_dim, (cudaStream_t)stream);
}

extern "C" int ymp_attn_fwd_prefix_kv(const ymp_attn_prefix_kv_args* c, void* stream) {
  using namespace ymp;
  YMP_CHECK_ARG(c != nullptr, "ymp_attn_fwd_prefix_kv: null args");
  AttnKParams p = {};
  const int rc = fill_table_params(&c->table, p, "ymp_attn_fwd_prefix_kv");
  if (rc) return rc;
  YMP_CHECK_ARG(c->k_cache && c->v_cache && aligned16(c->k_cache) && aligned16(c->v_cache),
                "ymp_attn_fwd_prefix_kv: k_cache / v_cache must be non-null and 16-byte aligned");
  YMP_CHECK_ARG(c->ld_cache % 8 == 0 && c->cache_head_stride % 8 == 0,
                "ymp_attn_fwd_prefix_kv: ld_cache and cache_head_stride must be multiples of 8");
  YMP_CHECK_ARG(c->n0 >= 0, "ymp_attn_fwd_prefix_kv: n0 must be >= 0");
  p.kc = (const __nv_bfloat16*)c->k_cache; p.vc = (const __nv_bfloat16*)c->v_cache;
  p.ldc = c->ld_cache; p.hsc = c->cache_head_stride; p.n0 = c->n0;
  g_attn_path = YMP_ATTN_PATH_WGMMA;
  return launch_wg_fwd_table<true>(p, c->table.attn.head_dim, (cudaStream_t)stream);
}

extern "C" int ymp_attn_fwd_packed(const ymp_attn_packed_args* a, void* stream) {
  using namespace ymp;
  const char* who = "ymp_attn_fwd_packed";
  YMP_CHECK_ARG(a != nullptr, "%s: null args", who);
  YMP_CHECK_ARG(a->starts != nullptr, "%s: null starts", who);
  YMP_CHECK_ARG(a->max_len >= 0, "%s: max_len must be >= 0", who);
  ymp_attn_args t = a->attn;
  t.s_q = t.s_kv = a->max_len > 0 ? a->max_len : 1;   // (only bounds the grid)
  AttnKParams p = {};
  const int rc = fill_params(&t, p, who);
  if (rc) return rc;
  YMP_CHECK_ARG(t.o && aligned16(t.o), "%s: bad o", who);
  YMP_CHECK_ARG(t.mask == YMP_MASK_CAUSAL, "%s: the mask must be causal", who);
  YMP_CHECK_ARG(t.head_dim != 128, "%s: needs head_dim 64, 80, 88 or 96", who);
  YMP_CHECK_ARG(!p.has_drop, "%s: takes no dropout", who);
  YMP_CHECK_ARG(!t.s_kv_dev, "%s: takes no s_kv_dev", who);
  YMP_CHECK_ARG(!t.kv_rows, "%s: takes no kv_rows", who);
  YMP_CHECK_ARG(t.total_rows == 0, "%s: takes no total_rows (starts gives every sequence's rows)", who);
  p.starts = a->starts;
  g_attn_path = YMP_ATTN_PATH_WGMMA;
  if (a->max_len == 0) return YMP_OK;   // every sequence is empty: nothing to write
  return launch_wg_fwd_packed(p, t.head_dim, (cudaStream_t)stream);
}

extern "C" int ymp_attn_bwd(const ymp_attn_bwd_args* b, void* stream) {
  using namespace ymp;
  YMP_CHECK_ARG(b != nullptr, "ymp_attn_bwd: null args");
  const ymp_attn_args* a = &b->fwd;
  AttnKParams p = {};
  int rc = fill_params(a, p, "ymp_attn_bwd");
  if (rc) return rc;
  YMP_CHECK_ARG(a->o && a->lse && b->dout && b->dq && b->dk && b->dv && b->delta_ws, "ymp_attn_bwd: null o/lse/dout/dq/dk/dv/delta_ws");
  YMP_CHECK_ARG(b->lddo % 8 == 0 && b->lddq % 8 == 0 && b->lddk % 8 == 0 && b->lddv % 8 == 0, "ymp_attn_bwd: grad row strides must be multiples of 8");
  YMP_CHECK_ARG(!a->s_kv_dev, "ymp_attn_bwd: s_kv_dev is forward only");
  YMP_CHECK_ARG(!a->kv_rows, "ymp_attn_bwd: kv_rows is forward only");
  YMP_CHECK_ARG(a->mask != YMP_MASK_CAUSAL || a->s_q == a->s_kv, "ymp_attn_bwd: causal with s_q < s_kv is forward only");
  YMP_CHECK_ARG(!p.has_drop || a->drop.p < 1.f, "ymp_attn_bwd: dropout p must be < 1");
  p.dout = (const __nv_bfloat16*)b->dout; p.dq = (__nv_bfloat16*)b->dq; p.dk = (__nv_bfloat16*)b->dk; p.dv = (__nv_bfloat16*)b->dv;
  p.delta = b->delta_ws;
  p.lddo = b->lddo; p.hsdo = b->do_head_stride;
  p.lddq = b->lddq; p.lddk = b->lddk; p.lddv = b->lddv;
  p.hsdq = b->dq_head_stride; p.hsdk = b->dk_head_stride; p.hsdv = b->dv_head_stride;
  p.mdo = to_map(b->map_do); p.mdq = to_map(b->map_dq); p.mdkv = to_map(b->map_dkv);
  cudaStream_t st = (cudaStream_t)stream;
  if (!p.has_drop) {
    rc = attn_small_bwd_try(b, st);
    if (rc != YMP_ENOSUP) { g_attn_path = YMP_ATTN_PATH_SMALL; return rc; }
  }
  if (a->head_dim != 128 && a->mask != YMP_MASK_BLOCK) {
    g_attn_path = YMP_ATTN_PATH_WGMMA;
    return launch_wg_bwd(p, a->head_dim, st);
  }
  g_attn_path = YMP_ATTN_PATH_MMA_SYNC;
  return launch_bwd(p, a->head_dim, st);
}
