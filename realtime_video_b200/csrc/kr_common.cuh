// kr_common.cuh — sm_90a PTX wrappers shared by every kernel in this library.
//
// Only inline PTX the Hopper programming model needs: mbarrier, TMA
// (cp.async.bulk.tensor), wgmma (fence / commit / wait, kr_wgmma.cuh) and the
// shared-memory matrix descriptors.  No CUTLASS / CuTe.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <stdint.h>

#include "../../include/krea_b200.h"
#include "kr_wgmma.cuh"

#define KR_DEVICE __device__ __forceinline__

namespace kr {

// ---------------------------------------------------------------------------
// error codes of the C ABI (include/krea_b200.h mirrors these)
// ---------------------------------------------------------------------------
// KR_OK / KR_ERR_* come from the public header

void set_last_error(const char* fmt, ...);

// ---------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------
KR_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
KR_DEVICE uint32_t lane_id() { return threadIdx.x & 31; }

KR_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------
KR_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
KR_DEVICE void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
KR_DEVICE void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
KR_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
KR_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
KR_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------
KR_DEVICE void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
KR_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
KR_DEVICE void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                           int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
KR_DEVICE void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                           int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
KR_DEVICE void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
KR_DEVICE void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
KR_DEVICE void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
KR_DEVICE void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA store / wgmma reads)
KR_DEVICE void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------------------
// clusters: rank, cluster-wide barrier, remote mbarrier arrive, multicast TMA
// ---------------------------------------------------------------------------
KR_DEVICE uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster (barrier init visible cluster-wide / no CTA exits while a peer may
// still multicast into its shared memory or arrive on its barriers)
KR_DEVICE void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster
KR_DEVICE void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [ra];\n\t}" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}
// the box lands at the same offset in every CTA of `mask`, each CTA's `bar` (same offset) receives the bytes
KR_DEVICE void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}

// ---------------------------------------------------------------------------
// wgmma (warpgroup MMA, accumulators in registers)
// ---------------------------------------------------------------------------
// Shared-memory matrix descriptor (64-bit), sm_90:
//   [0,14)  start address >> 4        [16,30) leading byte offset >> 4
//   [32,46) stride byte offset >> 4   [62,64) swizzle: 0 none, 1 SW128, 2 SW64, 3 SW32
// K-major SW128 operand: rows of 128 B (64 x 16-bit), 8-row groups 1024 B apart -> SBO = 1024, LBO unused;
//   the k-th 16-element step of a 64-wide panel starts 32 B further (the swizzle is applied to absolute
//   address bits, so tiles must be 1024-byte aligned).
// MN-major SW128 operand ([k][mn], 64 mn-elements = 128 B per k-row): 8 k-rows form a 1024 B atom; the next
//   8 k-rows are SBO bytes further, the next 64 mn-elements LBO bytes further.
enum : uint32_t { kSwz128 = 1, kSwz64 = 2, kSwz32 = 3 };
KR_DEVICE uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                  uint32_t swizzle = kSwz128) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(swizzle) << 62;
  return d;
}
KR_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
KR_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
KR_DEVICE void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keep the accumulator registers live and ordered around asynchronous wgmma (no code emitted)
template <int N>
KR_DEVICE void reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// register budget of a warpgroup (all its warps execute it): the TMA warpgroup gives registers back, the
// consumer warpgroups take them (3 warpgroups: 128 x 40 + 256 x 232 <= 64 K)
KR_DEVICE void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
KR_DEVICE void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }
// the same with another split (kernels whose producer warpgroup also runs an epilogue)
template <int R>
KR_DEVICE void producer_regs_n() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
KR_DEVICE void consumer_regs_n() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// named barrier over `count` threads (the consumer warpgroups of a kernel)
KR_DEVICE void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---------------------------------------------------------------------------
// numeric helpers
// ---------------------------------------------------------------------------
KR_DEVICE float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
KR_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
KR_DEVICE uint32_t pack_f16x2(float lo, float hi) {
  __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
KR_DEVICE float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
KR_DEVICE float2 unpack_f16x2(uint32_t u) {
  __half2 v = *reinterpret_cast<__half2*>(&u);
  return __half22float2(v);
}
KR_DEVICE float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// nn.GELU(approximate='tanh'), evaluated in fp32
KR_DEVICE float gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  float inner = k0 * (x + k1 * x * x * x);
  return 0.5f * x * (1.0f + tanhf(inner));
}

// ---------------------------------------------------------------------------
// host: TMA descriptor encode through the driver entry point (no -lcuda link)
// ---------------------------------------------------------------------------
// 2D row-major tensor [rows, cols] of 16-bit elements, row pitch in elements.
// box = [box_rows, box_cols]; swizzle 128B requires box_cols * 2 == 128.
int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                 uint64_t row_pitch_elems, uint32_t box_rows, uint32_t box_cols, bool is_bf16);
// generic N-d (<=5) map of 16-bit elements; dims/strides innermost first; strides in bytes
// for dims 1..n-1.
int make_tmap_nd(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box, bool is_bf16, int swizzle_bytes);

int make_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                 const uint32_t* box, int swizzle_bytes);

int sm_count();

}  // namespace kr
