// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma descriptors and fences.
// Everything here is architecture-specific on purpose: this library targets H100 only.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ymp {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* desc) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(desc)) : "memory");
}
// 2D tiled load global -> shared, completion signalled on mbarrier (complete_tx::bytes)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* desc, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)),
        "r"(c0), "r"(c1)
      : "memory");
}

// 5D tiled load (fused im2col of the patch embedding: coordinates {x, y, t, c, b} of a [B,C,T,H,W] video)
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const void* desc, uint64_t* bar, int32_t c0, int32_t c1,
                                            int32_t c2, int32_t c3, int32_t c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3), "r"(c4)
      : "memory");
}
// ---------------------------------------------------------------- wgmma (warpgroup MMA)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keep the accumulator registers ordered against the asynchronous wgmma that reads / writes them
template <int N>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor of wgmma (sm_90):
//   start address [0,14) >>4 | LBO [16,30) >>4 | SBO [32,46) >>4 | layout [62,64): 1 = SWIZZLE_128B, 3 = SWIZZLE_32B
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}

// ---------------------------------------------------------------- small math helpers
// programmatic dependent launch: wait until the preceding kernel of the stream has completed and its writes are visible
// (returns at once for an ordinary launch); allow the following kernel to start launching
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// streaming 128-bit load that does not allocate in L1 (weights read exactly once)
__device__ __forceinline__ uint4 ld_nc_v4(const uint4* p) {
  uint4 v;
  asm("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

// erf via Abramowitz-Stegun 7.1.26 (|abs err| < 1.5e-7: far below bf16 resolution)
__device__ __forceinline__ float fast_erf(float x) {
  float ax = fabsf(x);
  float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  float poly = fmaf(fmaf(fmaf(fmaf(1.061405429f, t, -1.453152027f), t, 1.421413741f), t,
                         -0.284496736f),
                    t, 0.254829592f) *
               t;
  float r = 1.0f - poly * __expf(-ax * ax);
  return copysignf(r, x);
}
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// exact-erf GELU (nn.GELU default) and its derivative, MUFU-light: Phi(x) = 0.5 + x Q(x^2) with a
// degree-9 near-minimax Q on |x| <= 4.5 (clamped outside; |Phi error| < 1e-5, |gelu error| < 5e-5, far
// below the bf16 resolution of the stored activation), the normal pdf by one MUFU.EX2.  18 issue slots per
// element instead of 28 + a MUFU.RCP: the K=768 ViT MLP GEMM epilogue stops being the bottleneck.
__device__ __forceinline__ float norm_cdf_pdf(float x, float& pdf) {
  const float xc = fminf(fmaxf(x, -4.5f), 4.5f);
  const float u = xc * xc;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fmaf(u, -0.72134752044f, -1.32574806474f)));
  pdf = e;  // exp(-x^2/2) / sqrt(2 pi)
  float q = -1.6543631001e-12f;
  q = fmaf(q, u, 1.9532824653e-10f);
  q = fmaf(q, u, -1.0287317553e-08f);
  q = fmaf(q, u, 3.2170341066e-07f);
  q = fmaf(q, u, -6.7323919166e-06f);
  q = fmaf(q, u, 1.0108823657e-04f);
  q = fmaf(q, u, -1.1397043329e-03f);
  q = fmaf(q, u, 9.8841767687e-03f);
  q = fmaf(q, u, -6.6411978624e-02f);
  q = fmaf(q, u, 3.9892175804e-01f);
  return fmaf(xc, q, 0.5f);  // Phi(x)
}
__device__ __forceinline__ float gelu_erf(float x) {
  float e;
  return x * norm_cdf_pdf(x, e);
}
// ---- fp32 pairs: two scalar IEEE operations each.  The GEMM epilogues are issue-slot / dependency-latency bound on the
// activation polynomials; the x8 helpers below interleave four independent chains.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 splat2(float c) { return make_float2(c, c); }

// Phi and the normal pdf of EIGHT values in lockstep (four packed pairs): the same arithmetic as norm_cdf_pdf, element
// by element, written coefficient-major so that the four dependency chains interleave.
__device__ __forceinline__ void norm_cdf_pdf_x8(const float (&x)[8], float2 (&cdf)[4], float2 (&pdf)[4]) {
  float2 xc[4], u[4], q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    xc[i] = make_float2(fminf(fmaxf(x[2 * i], -4.5f), 4.5f), fminf(fmaxf(x[2 * i + 1], -4.5f), 4.5f));
    u[i] = fmul2(xc[i], xc[i]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = ffma2(u[i], splat2(-0.72134752044f), splat2(-1.32574806474f));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(pdf[i].x) : "f"(a.x));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(pdf[i].y) : "f"(a.y));
    q[i] = ffma2(splat2(-1.6543631001e-12f), u[i], splat2(1.9532824653e-10f));
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = ffma2(q[i], u[i], splat2(-1.0287317553e-08f));
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = ffma2(q[i], u[i], splat2(3.2170341066e-07f));
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = ffma2(q[i], u[i], splat2(-6.7323919166e-06f));
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = ffma2(q[i], u[i], splat2(1.0108823657e-04f));
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = ffma2(q[i], u[i], splat2(-1.1397043329e-03f));
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = ffma2(q[i], u[i], splat2(9.8841767687e-03f));
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = ffma2(q[i], u[i], splat2(-6.6411978624e-02f));
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = ffma2(q[i], u[i], splat2(3.9892175804e-01f));
#pragma unroll
  for (int i = 0; i < 4; ++i) cdf[i] = ffma2(xc[i], q[i], splat2(0.5f));
}
// v = gelu_erf(x), d = gelu_erf'(x) for eight values (bit-identical to gelu_erf_both element by element)
__device__ __forceinline__ void gelu_erf_both_x8(const float (&x)[8], float (&v)[8], float (&d)[8]) {
  float2 cdf[4], pdf[4];
  norm_cdf_pdf_x8(x, cdf, pdf);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 xv = make_float2(x[2 * i], x[2 * i + 1]);
    const float2 dd = ffma2(xv, pdf[i], cdf[i]), vv = fmul2(xv, cdf[i]);
    d[2 * i] = dd.x; d[2 * i + 1] = dd.y; v[2 * i] = vv.x; v[2 * i + 1] = vv.y;
  }
}
__device__ __forceinline__ void gelu_erf_x8(const float (&x)[8], float (&v)[8]) {
  float2 cdf[4], pdf[4];
  norm_cdf_pdf_x8(x, cdf, pdf);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 vv = fmul2(make_float2(x[2 * i], x[2 * i + 1]), cdf[i]);
    v[2 * i] = vv.x; v[2 * i + 1] = vv.y;
  }
}
// GELU and its derivative together (the derivative is what backward needs; it is stored in bf16 by the
// forward epilogue so that the backward epilogue is a plain multiply)
__device__ __forceinline__ float gelu_erf_both(float x, float& d) {
  float e;
  const float cdf = norm_cdf_pdf(x, e);
  d = fmaf(x, e, cdf);
  return x * cdf;
}
__device__ __forceinline__ float gelu_tanh_both(float x, float& d) {
  const float u = 0.79788456f * x * fmaf(0.044715f * x, x, 1.0f);
  const float t = tanh_fast(u);
  const float du = 0.79788456f * fmaf(0.134145f * x, x, 1.0f);
  const float hp = 0.5f * (1.0f + t);
  d = fmaf(0.5f * x * (1.0f - t * t), du, hp);
  return x * hp;
}
__device__ __forceinline__ float dgelu_erf(float x) {
  float e;
  const float cdf = norm_cdf_pdf(x, e);
  return fmaf(x, e, cdf);
}
// tanh-approximation GELU (Megatron bias_gelu) and its derivative
__device__ __forceinline__ float gelu_tanh(float x) {
  float u = 0.79788456f * x * fmaf(0.044715f * x, x, 1.0f);
  return 0.5f * x * (1.0f + tanh_fast(u));
}
__device__ __forceinline__ float dgelu_tanh(float x) {
  float u = 0.79788456f * x * fmaf(0.044715f * x, x, 1.0f);
  float t = tanh_fast(u);
  float du = 0.79788456f * fmaf(0.134145f * x, x, 1.0f);
  return 0.5f * (1.0f + t) + 0.5f * x * (1.0f - t * t) * du;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace ymp
