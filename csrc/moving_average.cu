// Exponential moving average of the weights (--moving_average_decay), kept by the chief in an fp32 shadow arena of the
// parameter arena's layout.  TF's ExponentialMovingAverage with num_updates = global step:
//
//   d = min(D, (1 + g) / (10 + g))      in double, g = the epoch word (global step of the weights just committed)
//   m = (float)(1 - d)
//   s = s - (s - w) * m                 fp32, each operation rounded on its own (no FMA contraction, subnormals kept), so
//                                       a float32 numpy emulation reproduces every bit
//
//   moving_average   grid of num_sms() CTAs, grid-stride over the arena in float4 with a scalar tail (any length).  Reads
//                    the epoch word itself, so the captured step graph bakes in no step.  CTA 0 stores g into a device word:
//                    the step the shadow holds.  Optional output: the bf16 copy (round to nearest even, the rounding of the
//                    training shadow) of up to two [begin, end) ranges of the shadow, for the tensor-core operands of an
//                    evaluation pass.  Without weights (w == null) nothing is averaged: the call only writes that bf16 copy.
#include "common.cuh"
#include "host_utils.h"

namespace dm {

constexpr int MA_THREADS = 512;

struct MaArgs {
  float* shadow;
  const float* w;               // null: bf16 copy only
  long long numel;
  const uint32_t* epoch;
  double decay;
  uint32_t* step_out;           // null: not recorded
  __nv_bfloat16* bf16;          // null: no bf16 copy; else indexed like the arena
  long long r0b, r0e, r1b, r1e; // bf16 ranges (elements)
};

// s - (s - w) * m with three separately rounded operations.  Written in PTX without .ftz: the library builds with
// --use_fast_math, which would flush subnormal operands and results of __fsub_rn / __fmul_rn to zero, and the float32
// emulation keeps them.
DMNIST_DEVICE float ma_update(float s, float w, float m) {
  float d, p, r;
  asm("sub.rn.f32 %0, %1, %2;" : "=f"(d) : "f"(s), "f"(w));
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(p) : "f"(d), "f"(m));
  asm("sub.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(s), "f"(p));
  return r;
}

DMNIST_DEVICE bool ma_in(const MaArgs& a, long long i) { return (i >= a.r0b && i < a.r0e) || (i >= a.r1b && i < a.r1e); }

__global__ void __launch_bounds__(MA_THREADS) moving_average_kernel(const __grid_constant__ MaArgs a) {
  float m = 0.f;
  if (a.w != nullptr) {
    const uint32_t g = *a.epoch;
    const double r = (1.0 + (double)g) / (10.0 + (double)g);
    m = __double2float_rn(1.0 - (a.decay < r ? a.decay : r));
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.step_out != nullptr) *a.step_out = g;
  }
  const long long n4 = a.numel >> 2;
  const long long stride = (long long)gridDim.x * MA_THREADS;
  for (long long i = (long long)blockIdx.x * MA_THREADS + threadIdx.x; i < n4; i += stride) {
    float4 s = reinterpret_cast<const float4*>(a.shadow)[i];
    if (a.w != nullptr) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(a.w) + i);
      s.x = ma_update(s.x, w.x, m);
      s.y = ma_update(s.y, w.y, m);
      s.z = ma_update(s.z, w.z, m);
      s.w = ma_update(s.w, w.w, m);
      reinterpret_cast<float4*>(a.shadow)[i] = s;
    }
    // ranges are multiples of 4 (checked by the host): a float4 lies wholly inside or outside
    if (a.bf16 != nullptr && ma_in(a, 4 * i)) {
      uint2 o;
      o.x = pack_bf16x2(s.x, s.y);
      o.y = pack_bf16x2(s.z, s.w);
      reinterpret_cast<uint2*>(a.bf16)[i] = o;
    }
  }
  // tail: the last numel % 4 elements, one thread each (CTA 0)
  const long long t = 4 * n4 + (long long)blockIdx.x * MA_THREADS + threadIdx.x;
  if (t < a.numel) {
    float s = a.shadow[t];
    if (a.w != nullptr) {
      s = ma_update(s, a.w[t], m);
      a.shadow[t] = s;
    }
    if (a.bf16 != nullptr && ma_in(a, t)) a.bf16[t] = __float2bfloat16_rn(s);
  }
}

}  // namespace dm

extern "C" {

// shadow: fp32 arena of `numel` floats, updated in place from the weights `w` (null: only the bf16 copy is written);
// epoch: the u32 epoch word of the control block; decay: D, 0 < D < 1; step_out: u32 device word or null; bf16: arena-sized
// bf16 buffer or null, written on [r0b, r0e) and [r1b, r1e) (multiples of 4; empty ranges allowed).
int dm_moving_average(void* shadow, const void* w, long long numel, const void* epoch, double decay, void* step_out,
                      void* bf16, long long r0b, long long r0e, long long r1b, long long r1e, void* stream) {
  if (numel < 1 || shadow == nullptr || (w != nullptr && (epoch == nullptr || !(decay > 0.0 && decay < 1.0))) ||
      ((r0b | r0e | r1b | r1e) & 3) || r0b < 0 || r0e < r0b || r1b < 0 || r1e < r1b || r0e > numel || r1e > numel)
    return -1;
  dm::MaArgs a;
  a.shadow = reinterpret_cast<float*>(shadow);
  a.w = reinterpret_cast<const float*>(w);
  a.numel = numel;
  a.epoch = reinterpret_cast<const uint32_t*>(epoch);
  a.decay = decay;
  a.step_out = reinterpret_cast<uint32_t*>(step_out);
  a.bf16 = reinterpret_cast<__nv_bfloat16*>(bf16);
  a.r0b = r0b; a.r0e = r0e; a.r1b = r1b; a.r1e = r1e;
  const long long blocks = (numel / 4 + dm::MA_THREADS - 1) / dm::MA_THREADS;
  const int grid = blocks < 1 ? 1 : (blocks < dm::num_sms() ? (int)blocks : dm::num_sms());
  dm::moving_average_kernel<<<grid, dm::MA_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  return (int)cudaGetLastError();
}

}  // extern "C"
