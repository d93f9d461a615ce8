// Random affine augmentation of the training images (--augment_max_shift / _rotation / _scale), the first compute node
// of a training step: the input slot's fp32 images [B, 784] -> an engine-owned fp32 buffer [B, 784] that every reader of
// the step's training images reads instead.  The transform is defined once in distributedmnist_b200/augment.py:
//
//   draws   u_k = (hash_mix(hash_mix(seed_mix, i), 4 b + k) >> 8) * 2^-24, k = 0..3, for row b at iteration i
//   theta = R pi/180 (2 u0 - 1)   s = 1 + S (2 u1 - 1)   tx = T (2 u2 - 1)   ty = T (2 u3 - 1)
//   a = cos(theta) / s, b = sin(theta) / s   (double, rounded once to fp32; one thread per row)
//   output pixel (x, y) samples the source bilinearly at, around c = 13.5,
//     sx = c + a dx + b dy,  sy = c - b dx + a dy,  dx = x - c - tx,  dy = y - c - ty
//   and a tap outside [0, 27]^2 reads the background -0.5 (a zero pixel after data.py's scaling).
//
// The coordinates and the blend are explicit single-rounding fmas (fma_rn: --use_fast_math must not flush or contract
// them differently), so the result does not depend on the compiler's choices.
//
// The iteration i is a u32 word on the device, counter[0]: every CTA reads it before it arrives on counter[1] (a ticket,
// see arrive_last_cta), and the last CTA to arrive stores i + 1.  A captured step graph so draws new numbers on every
// replay with no host value baked in.  One launch per counter in flight.
//
// CTA = AUG_THREADS threads over rows blockIdx.x, blockIdx.x + gridDim.x, ... (at most AUG_MAX_ROWS): thread t first
// computes the coefficients of the CTA's row t, then the CTA stages each row in shared memory and writes its 784 pixels.
#include "augment.cuh"
#include "host_utils.h"

namespace dm {

__global__ void __launch_bounds__(AUG_THREADS) augment_affine_kernel(const float* __restrict__ src,
                                                                     float* __restrict__ dst, int batch,
                                                                     unsigned int* counter, uint32_t seed_mix,
                                                                     AugRange rg, float* __restrict__ params_out) {
  __shared__ __align__(16) float s_img[AUG_PIX];
  __shared__ float4 s_coef[AUG_MAX_ROWS];
  __shared__ unsigned int s_flag;
  pdl_wait();                               // the previous step's readers of dst are done; the slot's copy has landed
  const int nrows = (batch - 1 - (int)blockIdx.x) / (int)gridDim.x + 1;
  const int t = threadIdx.x;
  if (t < nrows) {
    const uint32_t it = __ldcg(counter);    // read before this CTA arrives on the ticket
    const int b = (int)blockIdx.x + t * (int)gridDim.x;
    s_coef[t] = affine_row_coefficients(hash_mix(seed_mix, it), b, rg, params_out);
  }
  for (int r = 0; r < nrows; ++r) {
    const size_t row = (size_t)((int)blockIdx.x + r * (int)gridDim.x) * AUG_PIX;
    __syncthreads();                        // s_coef complete (r = 0); every thread is done with the previous row
    if (t < AUG_PIX / 4)
      reinterpret_cast<float4*>(s_img)[t] = __ldg(reinterpret_cast<const float4*>(src + row) + t);
    __syncthreads();
    const float4 c = s_coef[r];
    for (int p = t; p < AUG_PIX; p += AUG_THREADS) {
      const int y = p / 28, x = p - 28 * y;
      const float dx = ((float)x - 13.5f) - c.z;      // x - 13.5 is exact: one rounding
      const float dy = ((float)y - 13.5f) - c.w;
      // far outside the image every tap is background: clamping there changes nothing and keeps the floor in int range
      const float sx = fminf(fmaxf(fma_rn(c.x, dx, fma_rn(c.y, dy, 13.5f)), -2.f), 29.f);
      const float sy = fminf(fmaxf(fma_rn(c.x, dy, fma_rn(-c.y, dx, 13.5f)), -2.f), 29.f);
      const float fx0 = floorf(sx), fy0 = floorf(sy);
      const float fx = sx - fx0, fy = sy - fy0;          // exact
      const int x0 = (int)fx0, y0 = (int)fy0;
      const bool cx0 = (unsigned)x0 < 28u, cx1 = (unsigned)(x0 + 1) < 28u;
      const bool cy0 = (unsigned)y0 < 28u, cy1 = (unsigned)(y0 + 1) < 28u;
      const float v00 = cy0 && cx0 ? s_img[y0 * 28 + x0] : -0.5f;
      const float v01 = cy0 && cx1 ? s_img[y0 * 28 + x0 + 1] : -0.5f;
      const float v10 = cy1 && cx0 ? s_img[(y0 + 1) * 28 + x0] : -0.5f;
      const float v11 = cy1 && cx1 ? s_img[(y0 + 1) * 28 + x0 + 1] : -0.5f;
      const float top = fma_rn(fx, v01 - v00, v00);
      const float bot = fma_rn(fx, v11 - v10, v10);
      dst[row + p] = fma_rn(fy, bot - top, top);
    }
  }
  if (arrive_last_cta(counter + 1, gridDim.x, 1, AUG_THREADS, &s_flag) && t == 0) counter[0] = __ldcg(counter) + 1u;
}

}  // namespace dm

extern "C" {

// src, dst: fp32 [batch, 784] (device memory, 16-byte aligned, not overlapping); counter: two u32 words of device memory,
// the iteration and a ticket that must be 0 between launches (each launch leaves it 0); seed_mix: augment.seed_mix(seed,
// rank); max_shift, max_rotation (degrees), max_scale: finite, >= 0, max_scale < 1.  params_out: null, or batch * 8 floats
// receiving each row's u0..u3 and the a, b, tx, ty it used.  Enqueued on `stream`; advances counter[0] by one.
int dm_augment_affine(const void* src, void* dst, int batch, void* counter, unsigned int seed_mix, double max_shift,
                      double max_rotation, double max_scale, void* params_out, void* stream) {
  using namespace dm;
  if (src == nullptr || dst == nullptr || counter == nullptr || batch < 1) return -1;
  if (!(isfinite(max_shift) && isfinite(max_rotation) && isfinite(max_scale)) || max_shift < 0.0 || max_rotation < 0.0 ||
      max_scale < 0.0 || max_scale >= 1.0)
    return -1;
  const int grid = augment_grid(batch, num_sms());
  const AugRange rg{max_shift, max_rotation, max_scale};
  return (int)launch_kernel(augment_affine_kernel, dim3(grid), dim3(AUG_THREADS), 0, reinterpret_cast<cudaStream_t>(stream),
                            reinterpret_cast<const float*>(src), reinterpret_cast<float*>(dst), batch,
                            reinterpret_cast<unsigned int*>(counter), (uint32_t)seed_mix, rg,
                            reinterpret_cast<float*>(params_out));
}

}  // extern "C"
