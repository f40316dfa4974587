// Shared device helpers for the sm_90a kernels of omnidata_b200.
// Thin inline-PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor); the wgmma wrappers are in wgmma.cuh.
// Nothing here is reference-derived; the reference (EPFL-VILAB/omnidata) has no native code on this path.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define ODB_DEVINL __device__ __forceinline__

namespace odb {

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------- shared-memory addressing
ODB_DEVINL uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
ODB_DEVINL void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
ODB_DEVINL void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
ODB_DEVINL void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
ODB_DEVINL void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
ODB_DEVINL bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin with a watchdog: a protocol bug must abort the kernel (sticky error on the host)
// instead of hanging the GPU.  Trap only, no printf: a printf is a function call, and a call
// inlined between wgmma issue and wait makes ptxas serialise every wgmma of the kernel (C7510).
ODB_DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}

// ---------------------------------------------------------------- programmatic dependent launch
// Every forward-path kernel is launched with programmaticStreamSerialization: it may start (and run
// its prologue: barrier init, descriptor prefetch) while the previous kernel of the
// stream drains.  grid_dep_wait() must precede the first access to global memory.
ODB_DEVINL void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
ODB_DEVINL void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- fences / named barriers
ODB_DEVINL void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
ODB_DEVINL void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- TMA
ODB_DEVINL void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
ODB_DEVINL void tma_load_2d(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar, int c0,
                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4}], [%2];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
ODB_DEVINL void tma_load_4d(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar, int c0,
                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
ODB_DEVINL void tma_store_4d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1, int c2,
                             int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(map)),
      "r"(smem_src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// the same box written to the same shared-memory offset of every CTA in `cta_mask` (a cluster); each destination
// CTA's mbarrier at offset `bar` receives the complete_tx of the bytes it got
ODB_DEVINL void tma_load_2d_multicast(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar, int c0, int c1,
                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster "
      "[%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}

// ---------------------------------------------------------------- clusters
ODB_DEVINL uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
ODB_DEVINL void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cta address of this CTA -> shared::cluster address of the same offset in CTA `rank`
ODB_DEVINL uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
ODB_DEVINL void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}

ODB_DEVINL void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
ODB_DEVINL void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
ODB_DEVINL void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------- small numerics helpers
// erf via Abramowitz-Stegun 7.1.26 (|abs err| < 1.5e-7, far below one bf16 ulp of the GELU output):
// 1 MUFU.RCP + 1 MUFU.EX2 + 9 FMA-class ops instead of the ~30-instruction libdevice erff.
ODB_DEVINL float erf_as(float x) {
  const float ax = fabsf(x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = __expf(-ax * ax);
  return copysignf(fmaf(-p * t, e, 1.0f), x);
}
ODB_DEVINL float gelu_erf(float x) { return 0.5f * x * (1.0f + erf_as(x * 0.70710678118654752f)); }

ODB_DEVINL float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// Exact-erf GELU for the GEMM epilogue, two elements at a time:
//   gelu(x) = x Phi(x) = max(x, 0) - |x| Phi(-|x|),   Phi(-a) = 2^P(a),  a = min(|x|, 8)
// P = degree-10 weighted-minimax fit of log2 Phi(-a) on [0, 8] (fit: |gelu error| < 4e-8 absolute AND
// < 6e-6 relative — the tail x -> -inf keeps RELATIVE accuracy because the error sits in the
// exponent; measured in fp32 against float64 x Phi(x): 2.4e-7 = half an ulp of the result).
// Cost per element: 10 FFMA + 1 MUFU.EX2 + 3 ALU — half the MUFU work of the Abramowitz-Stegun form above,
// which is what bounds the fc1 epilogue (16 MUFU results per clock per SM).
ODB_DEVINL void gelu_erf_x2(float& x0, float& x1) {
  const float a0 = fminf(fabsf(x0), 8.0f), a1 = fminf(fabsf(x1), 8.0f);
  constexpr float kC[11] = {-4.45074694e-09f, 1.77394618e-07f, -2.91884744e-06f, 2.41618334e-05f, -7.56097581e-05f,
                            -4.90890656e-04f, 7.66879548e-03f,  -5.30659795e-02f, -4.58926226e-01f, -1.15116936e+00f,
                            -9.99995267e-01f};
  float p0 = fmaf(kC[0], a0, kC[1]), p1 = fmaf(kC[0], a1, kC[1]);
#pragma unroll
  for (int i = 2; i < 11; ++i) {
    p0 = fmaf(p0, a0, kC[i]);
    p1 = fmaf(p1, a1, kC[i]);
  }
  x0 = fmaf(-a0, ex2_approx(p0), fmaxf(x0, 0.0f));
  x1 = fmaf(-a1, ex2_approx(p1), fmaxf(x1, 0.0f));
}

ODB_DEVINL uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
ODB_DEVINL float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

ODB_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
ODB_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- ordered reduction of per-block partials (256-thread blocks)
// Block = 32 adjacent columns x 8 part lanes: lane l sums parts l, l+8, ... in fp64 (independent loads, four in flight),
// then the lane-0 threads add the 8 lane sums in lane order.  The order is fixed for a given `parts`, so results are
// bit-reproducible, and the dependent chain is parts / 8 long instead of parts.  The value is returned to the threads
// of part lane 0 (threadIdx.x < 32).
template <typename F>
ODB_DEVINL double ordered_sum8(int parts, bool active, F&& part) {
  __shared__ double sh_os8[8][33];
  const int col = threadIdx.x & 31, pl = threadIdx.x >> 5;
  double t = 0.0;
  if (active) {
#pragma unroll 4
    for (int p = pl; p < parts; p += 8) t += (double)part(p);
  }
  sh_os8[pl][col] = t;
  __syncthreads();
  double s = 0.0;
  if (pl == 0) {
#pragma unroll
    for (int l = 0; l < 8; ++l) s += sh_os8[l][col];
  }
  return s;
}


}  // namespace odb
