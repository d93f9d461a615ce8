// The per-row affine coefficients of the training-image augmentation (distributedmnist_b200/augment.py), shared by
// augment_affine (augment.cu) and augment_elastic (augment_elastic.cu) so that both compute them bit for bit alike.
#pragma once

#include <math.h>

#include "common.cuh"

namespace dm {

constexpr int AUG_THREADS = 256;
constexpr int AUG_MAX_ROWS = 32;          // rows per CTA; the grid grows past 4 CTAs per SM beyond that
constexpr int AUG_PIX = 784;
constexpr int AUG_PARAMS = 8;             // params_out per row: u0..u3, a, b, tx, ty

struct AugRange {
  double max_shift, max_rotation, max_scale;   // T (pixels), R (degrees), S
};

// Row b's draws u0..u3 under key = hash_mix(seed_mix, i) and its (a, b, tx, ty): double, each rounded once to fp32.
// Writes the eight params_out words of the row when params_out is not null.
__device__ __forceinline__ float4 affine_row_coefficients(uint32_t key, int b, const AugRange& rg,
                                                          float* __restrict__ params_out) {
  float u[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) u[k] = (float)(hash_mix(key, 4u * (uint32_t)b + (uint32_t)k) >> 8) * 0x1p-24f;
  const double theta = rg.max_rotation * M_PI / 180.0 * (2.0 * (double)u[0] - 1.0);
  const double s = 1.0 + rg.max_scale * (2.0 * (double)u[1] - 1.0);
  double sn, cs;
  sincos(theta, &sn, &cs);
  const float4 c = make_float4(__double2float_rn(cs / s), __double2float_rn(sn / s),
                               __double2float_rn(rg.max_shift * (2.0 * (double)u[2] - 1.0)),
                               __double2float_rn(rg.max_shift * (2.0 * (double)u[3] - 1.0)));
  if (params_out != nullptr) {
    float* p = params_out + (size_t)b * AUG_PARAMS;
    p[0] = u[0]; p[1] = u[1]; p[2] = u[2]; p[3] = u[3];
    p[4] = c.x; p[5] = c.y; p[6] = c.z; p[7] = c.w;
  }
  return c;
}

// The grid of both augmentation kernels: min(4 CTAs per SM, batch), grown to ceil(batch / AUG_MAX_ROWS) when that is more.
inline int augment_grid(int batch, int sms) {
  int grid = 4 * sms;
  if (grid > batch) grid = batch;
  if (grid < (batch + AUG_MAX_ROWS - 1) / AUG_MAX_ROWS) grid = (batch + AUG_MAX_ROWS - 1) / AUG_MAX_ROWS;
  return grid;
}

}  // namespace dm
