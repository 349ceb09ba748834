// Thin inline-PTX wrappers for the sm_90a features the kernels use: mbarrier, bulk async copy (UBLKCP) and tensor copy
// (TMA), the warpgroup MMA (wgmma) fences and the shared-memory matrix descriptors.
// Every spin-wait is BOUNDED: a wait that does not complete traps (kernel error) instead of hanging the GPU.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "wgmma.cuh"

namespace nero {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// volatile keeps the store ahead of the fence / barrier that publishes it
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v));
}
// the same store, executed only where `on` holds (a predicated instruction, not a branch)
__device__ __forceinline__ void sts_u32_if(uint32_t addr, uint32_t v, bool on) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p st.shared.b32 [%0], %1;\n\t}" ::"r"(addr), "r"(v), "r"(uint32_t(on)));
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: ~2^24 polls (a few seconds) then trap -> the launch fails loudly instead of hanging the GPU.  (No printf
// here: a function call inside the wgmma pipeline makes ptxas serialise every wgmma of the kernel.)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) __trap();
  }
}
// The same bounded wait for code that keeps wgmma groups in flight across it: a trap there makes ptxas retire every
// wgmma before the wait (C7517, "warpgroup.wait is injected").  A wait that does not complete sets `timed_out` and
// returns instead; the caller traps once its MMAs have drained.
__device__ __forceinline__ void mbar_wait_flag(uint64_t* bar, uint32_t parity, bool& timed_out) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 24)) {
      timed_out = true;
      return;
    }
  }
}

// make generic-proxy smem writes visible to the async proxy (wgmma / bulk copies read smem through it)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// shared-memory counter: adds v and returns the old value, with acquire-release ordering at CTA scope (the accesses
// ordered before one thread's add are visible to a thread whose later add reads its result)
__device__ __forceinline__ uint32_t atom_add_acq_rel_smem(uint32_t addr, uint32_t v) {
  uint32_t old;
  asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(addr), "r"(v) : "memory");
  return old;
}
// named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ------------------------------------------------------------------ L2 cache policies (per-instruction hints)
// lines an access with this policy brings into L2 are evicted after normal and evict-first lines
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// ------------------------------------------------------------------ bulk async copy global -> shared (UBLKCP)
// with the L2 policy `l2_policy` (createpolicy) for the source lines
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar, uint64_t l2_policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(l2_policy)
      : "memory");
}

// 2-D tensor copy (TMA) of the box at coordinates (c0 = innermost, c1) of `tmap` (a __grid_constant__ kernel parameter);
// elements outside the tensor arrive as zeros and count towards the transaction bytes
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}

// ------------------------------------------------------------------ per-thread async copy global -> shared (LDGSTS)
// 16 bytes; the first src_bytes (0..16) come from gmem_src (16-byte aligned), the rest is zero-filled.  Through L2 only (.cg).
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void* gmem_src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gmem_src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// the thread's own copies of all but the newest N committed groups have landed (and are visible to it)
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ------------------------------------------------------------------ wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}

// ------------------------------------------------------------------ descriptors (sm_90 GMMA layout)
// start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout [62,64): 1 = SWIZZLE_128B
// K-major operand tile, 128-byte swizzle: rows are 128 B (64 bf16) apart, 8-row groups 1024 B apart (LBO unused).
__device__ __forceinline__ uint64_t make_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// K-major operand tile, 64-byte swizzle: rows are 64 B (32 bf16) apart, 8-row groups 512 B apart (LBO unused).
__device__ __forceinline__ uint64_t make_desc_k_sw64(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(512 >> 4) << 32;
  d |= static_cast<uint64_t>(2) << 62;
  return d;
}
// MN-major operand tile, 128-byte swizzle (canonical layout ((8,8,m),(8,k)):((1,8,LBO),(64,SBO)) in bf16 elements): an
// atom is 8 K-rows x 64 MN-elements (8 x 128 B, 16-byte chunks XOR-swizzled with the row index); atoms repeat along MN
// every `lbo` bytes and along K every `sbo` bytes.
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo >> 4) << 16;
  d |= static_cast<uint64_t>(sbo >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

}  // namespace nero
