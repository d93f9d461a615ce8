// Shared device-side building blocks for the sm_90a kernels: mbarrier, TMA, ldmatrix,
// wgmma wrappers, wgmma descriptor encoder, small math helpers.
//
// Everything here is written directly against the PTX ISA for sm_90a (no CUTLASS
// dependency); the bit layout of the shared-memory matrix descriptor follows the PTX
// "wgmma matrix descriptor" table.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define DMNIST_DEVICE __device__ __forceinline__

namespace dm {

// ---------------------------------------------------------------------------------
// misc
// ---------------------------------------------------------------------------------
DMNIST_DEVICE uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
DMNIST_DEVICE uint32_t lane_id() { return threadIdx.x & 31; }

DMNIST_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// Counter-based hash: murmur3's 32-bit finaliser over idx * golden ratio + seed_mix.
DMNIST_DEVICE uint32_t hash_mix(uint32_t seed_mix, uint32_t idx) {
  uint32_t x = idx * 0x9E3779B1u + seed_mix;
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return x;
}

// Counter-based dropout: identical to models/lenet.py::dropout_keep_mask.
DMNIST_DEVICE bool dropout_keep(uint32_t seed_mix, uint32_t idx, uint32_t thresh24) {
  return (hash_mix(seed_mix, idx) >> 8) < thresh24;
}

DMNIST_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// prmt.b32, generic mode: result byte i = byte (sel nibble i & 7) of {b:a}; nibble bit 3 set -> the selected byte's
// sign bit replicated over the result byte (0x00 / 0xff): turns per-byte flags into lane masks.
DMNIST_DEVICE uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}

// 16-byte vector reduction into global memory (sm_90+): one instruction adds four consecutive floats.
DMNIST_DEVICE void red_add_f32x4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// a * b + c with one rounding, subnormals kept: written in PTX because --use_fast_math turns fmaf into fma.rn.ftz, and
// the L2 decay epilogues must equal an exact single-rounding emulation
DMNIST_DEVICE float fma_rn(float a, float b, float c) {
  float d;
  asm("fma.rn.f32 %0, %1, %2, %3;" : "=f"(d) : "f"(a), "f"(b), "f"(c));
  return d;
}

DMNIST_DEVICE uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---------------------------------------------------------------------------------
// programmatic dependent launch
// ---------------------------------------------------------------------------------
// Block until every kernel this launch depends on has completed and its writes are visible
// (no-op when the kernel was launched without the PDL attribute).
DMNIST_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// Allow the dependent kernel's CTAs to be scheduled (they still block in their own pdl_wait()).
DMNIST_DEVICE void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------
DMNIST_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
DMNIST_DEVICE void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
DMNIST_DEVICE void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

DMNIST_DEVICE void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
DMNIST_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
DMNIST_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
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
DMNIST_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor), completion on an mbarrier
// ---------------------------------------------------------------------------------
DMNIST_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
DMNIST_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
DMNIST_DEVICE void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                               int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// ---------------------------------------------------------------------------------
// ldmatrix: 8x8 b16 tiles from shared memory into the mma / wgmma register-fragment layout
// ---------------------------------------------------------------------------------
// Lane l supplies the row address of tile l / 8 (row l % 8).  Register i of every lane holds tile i:
// without .trans lane l gets row l / 4, elements 2 (l % 4) and 2 (l % 4) + 1; with .trans the tile is read
// column-wise (lane l gets column l / 4, rows 2 (l % 4) and 2 (l % 4) + 1).
DMNIST_DEVICE void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
DMNIST_DEVICE void ldsm_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}

// ---------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 in, fp32 accumulate in registers
// ---------------------------------------------------------------------------------
// Accumulator layout (per warp w of the warpgroup, lane l, g = l / 4, t = l % 4):
//   d[4 j + 0], d[4 j + 1] = row 16 w + g,     columns 8 j + 2 t, 8 j + 2 t + 1
//   d[4 j + 2], d[4 j + 3] = row 16 w + g + 8, same columns
// A from registers uses the m16n8k16 A-fragment layout for the warp's 16 rows (what ldsm_x4 delivers for
// tiles {rows 0-7, k 0-7}, {rows 8-15, k 0-7}, {rows 0-7, k 8-15}, {rows 8-15, k 8-15}).
DMNIST_DEVICE void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
DMNIST_DEVICE void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
DMNIST_DEVICE void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
DMNIST_DEVICE void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// A and B from shared-memory descriptors; TA / TB = 1: operand is MN-major.
template <int TA, int TB>
DMNIST_DEVICE void wgmma_m64n64_ss(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}
template <int TA, int TB>
DMNIST_DEVICE void wgmma_m64n128_ss(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TA), "n"(TB)
      : "memory");
}
// A from registers, B from a shared-memory descriptor.
template <int TB>
DMNIST_DEVICE void wgmma_m64n64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate), "n"(TB)
      : "memory");
}
template <int TB>
DMNIST_DEVICE void wgmma_m64n32_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, %22;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate), "n"(TB)
      : "memory");
}

// Named barrier over the first `threads` threads of the CTA (id 0 is __syncthreads).
DMNIST_DEVICE void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---------------------------------------------------------------------------------
// deterministic cross-CTA reductions
// ---------------------------------------------------------------------------------
// Every CTA stores its partial sums to its own slot of a global workspace and then takes a ticket; the CTA that draws
// the last ticket (returns true in all its threads) adds the slots up in slot order.  Unlike atomics into the output,
// the summation order -- and so the result, to the bit -- does not depend on which CTA finishes first.
// The workspaces and tickets are static per device (one set per kernel), so each of these kernels may have only ONE
// launch in flight per device: launches on the same stream (the training step) are fine, concurrent launches of the
// same kernel on two streams would mix their partial sums.  `threads` =
// the CTA threads taking part (they must include thread 0), `bar_id` a named barrier reserved for them.  The last CTA
// resets the ticket for the next launch.
DMNIST_DEVICE bool arrive_last_cta(unsigned int* ticket, unsigned int ctas, uint32_t bar_id, uint32_t threads,
                                   volatile unsigned int* s_flag) {
  __threadfence();                                  // this CTA's partial is visible before its ticket
  named_bar_sync(bar_id, threads);
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(ticket, 1u);
    *s_flag = (t == ctas - 1) ? 1u : 0u;
    if (t == ctas - 1) *ticket = 0u;
  }
  named_bar_sync(bar_id, threads);
  const bool last = *s_flag != 0u;
  if (last) __threadfence();                        // acquire side: the other CTAs' partials (read with __ldcg)
  return last;
}

// sum_{k < n} p[k * stride] in k order, float4-wide; 16 loads in flight (L2, bypassing L1) per round.
DMNIST_DEVICE float4 ordered_sum4(const float4* p, int n, size_t stride) {
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k0 = 0; k0 < n; k0 += 16) {
    float4 v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) v[u] = k0 + u < n ? __ldcg(p + (size_t)(k0 + u) * stride) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int u = 0; u < 16; ++u)
      if (k0 + u < n) { s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w; }
  }
  return s;
}

// out[4q .. 4q + 3] += columns 4q .. 4q + 3 of sum_{k < n} slots[k][0..63], each column added in slot order from zero.
// The NT threads of the CTA copy 4 NT slots' float4 at a time into s_buf, all loads in flight together (one L2 round
// trip per 4 NT slots), and thread 0 adds them.
template <int NT>
DMNIST_DEVICE void add_ordered_slot_sum64(const float* slots, int n, int q, float* out, float4 (&s_buf)[4 * NT]) {
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* src = reinterpret_cast<const float4*>(slots) + q;
  for (int k0 = 0; k0 < n; k0 += 4 * NT) {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int k = k0 + u * NT + (int)threadIdx.x;
      if (k < n) v[u] = __ldcg(src + (size_t)k * 16);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (k0 + u * NT + (int)threadIdx.x < n) s_buf[u * NT + threadIdx.x] = v[u];
    __syncthreads();
    if (threadIdx.x == 0) {
      const int m = min(4 * NT, n - k0);
      for (int k = 0; k < m; ++k) { s.x += s_buf[k].x; s.y += s_buf[k].y; s.z += s_buf[k].z; s.w += s_buf[k].w; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float4* o = reinterpret_cast<float4*>(out) + q;
    const float4 cur = *o;
    *o = make_float4(cur.x + s.x, cur.y + s.y, cur.z + s.z, cur.w + s.w);
  }
}

// ---------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptors
// ---------------------------------------------------------------------------------
enum : uint32_t { SWZ_NONE = 0, SWZ_128B = 1, SWZ_64B = 2, SWZ_32B = 3 };

// Shared-memory matrix descriptor (64 bit, sm_90):
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4   [49,52) base offset (0: tiles are aligned to the swizzle repeat)
//   [62,64) swizzle mode
// K-major operand, swizzled:   rows of <swizzle width> bytes, 8-row groups SBO apart (LBO unused); a K step
//                              inside the swizzle width advances the start address.
// MN-major operand, swizzled:  k-rows of <swizzle width> bytes; 8-k groups SBO apart; successive
//                              <swizzle width> chunks along M/N are LBO apart.
DMNIST_DEVICE uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t swizzle) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)(swizzle & 3) << 62;
  return d;
}
// Advance the start address of a descriptor by `bytes` (stays inside the 14-bit field:
// shared memory is < 256 KB so no carry into the LBO field can occur).
DMNIST_DEVICE uint64_t desc_advance(uint64_t desc, uint32_t bytes) { return desc + (uint64_t)(bytes >> 4); }

}  // namespace dm
