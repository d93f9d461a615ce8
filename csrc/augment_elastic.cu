// Elastic distortion of the training images (--augment_elastic_alpha / _sigma), composed with the random affine warp of
// augment.cu: with alpha > 0 this kernel takes augment_affine's place as the first compute node of a training step, reads
// the same input slot, writes the same engine-owned buffer and advances the same iteration counter.  The transform is
// defined once in distributedmnist_b200/augment.py:
//
//   affine  a, b, tx, ty of row b at iteration i: augment_affine's (affine_row_coefficients, bit for bit)
//   draws   v = 2 u - 1, u = (hash_mix(hash_mix(E, i), 1568 b + 784 d + p) >> 8) * 2^-24, E = seed_mix + ELASTIC_MIX,
//           d = 0 (x component) or 1 (y), p = 28 y + x: exact in fp32
//   field   e_d = alpha * G V_d G^T, G the normalised Gaussian of radius R <= 32 (taps outside the image read 0)
//   warp    output pixel (x, y) samples the source bilinearly at, around c = 13.5,
//             sx = c + a dx + b dy,  sy = c - b dx + a dy,  dx = (x - c + ex) - tx,  dy = (y - c + ey) - ty
//           and a tap outside [0, 27]^2 reads the background -0.5.
//
// Arithmetic.  The taps w_0..w_R are float64 values computed on the host (augment.gaussian_weights); the device
// evaluates no exp.  The field is two passes in double over the row's draws in shared memory: horizontal
// h = sum_k w_|k| v(x + k), then vertical s = sum_k w_|k| h(y + k), each an fma chain over k ascending from the first tap
// inside the image, then e = fl32(alpha * s).  Each pass adds at most (2R + 2) double roundings of terms whose magnitudes
// sum to <= 1 (|v| <= 1, sum w = 1), so |s - exact| <= 2 * 66 * 2^-53 < 2^-45 and e is the fp32 rounding of a value
// within alpha 2^-45 of the exact field: within one fp32 ulp of it, plus alpha 2^-45 where the field nearly cancels.
// The coordinates and the blend are explicit single-rounding operations (__fadd_rn, fma_rn: --use_fast_math must not
// contract them differently), in the order written above: xc = x - 13.5 (exact), fl(fl(xc + ex) - tx), then the fmas
// of augment_affine.  With ex = ey = 0 the coordinates are augment_affine's exactly.
//
// Counter protocol, grid and row striding are augment_affine's: counter[0] is the iteration, read by every CTA before it
// arrives on the ticket counter[1]; the last CTA to arrive stores i + 1.  One CTA works on one row at a time.
#include "augment.cuh"
#include "host_utils.h"

namespace dm {

constexpr int ELASTIC_MAX_RADIUS = 32;
constexpr int ELASTIC_DRAWS = 2 * AUG_PIX;          // per row: the x component's 784 draws, then the y component's
constexpr uint32_t ELASTIC_MIX = 0x6A09E667u;       // augment.ELASTIC_MIX
constexpr int ELASTIC_MAX_BATCH = 2739137;          // floor(2^32 / 1568): every draw index fits in u32

struct ElasticArgs {
  double alpha;
  int radius;
  double w[ELASTIC_MAX_RADIUS + 1];                 // w_0 .. w_radius; the rest unused
};

__global__ void __launch_bounds__(AUG_THREADS) augment_elastic_kernel(const float* __restrict__ src,
                                                                      float* __restrict__ dst, int batch,
                                                                      unsigned int* counter, uint32_t seed_mix,
                                                                      AugRange rg, ElasticArgs ea,
                                                                      float* __restrict__ params_out,
                                                                      float* __restrict__ field_out) {
  __shared__ __align__(16) float s_img[AUG_PIX];
  __shared__ float s_v[ELASTIC_DRAWS];
  __shared__ double s_h[ELASTIC_DRAWS];
  __shared__ double s_w[ELASTIC_MAX_RADIUS + 1];
  __shared__ float4 s_coef[AUG_MAX_ROWS];
  __shared__ unsigned int s_flag;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k <= ELASTIC_MAX_RADIUS; ++k) s_w[k] = ea.w[k];     // static indices: no local copy of the params
  }
  pdl_wait();                               // the previous step's readers of dst are done; the slot's copy has landed
  const int nrows = (batch - 1 - (int)blockIdx.x) / (int)gridDim.x + 1;
  const int t = threadIdx.x;
  const uint32_t it = __ldcg(counter);      // read before this CTA arrives on the ticket
  if (t < nrows) s_coef[t] = affine_row_coefficients(hash_mix(seed_mix, it), (int)blockIdx.x + t * (int)gridDim.x, rg,
                                                     params_out);
  const uint32_t ekey = hash_mix(seed_mix + ELASTIC_MIX, it);
  const int R = ea.radius;
  for (int r = 0; r < nrows; ++r) {
    const int b = (int)blockIdx.x + r * (int)gridDim.x;
    const size_t row = (size_t)b * AUG_PIX;
    __syncthreads();                        // s_coef, s_w complete (r = 0); every thread is done with the previous row
    if (t < AUG_PIX / 4)
      reinterpret_cast<float4*>(s_img)[t] = __ldg(reinterpret_cast<const float4*>(src + row) + t);
    for (int j = t; j < ELASTIC_DRAWS; j += AUG_THREADS)
      s_v[j] = (float)(hash_mix(ekey, (uint32_t)ELASTIC_DRAWS * (uint32_t)b + (uint32_t)j) >> 8) * 0x1p-23f - 1.0f;
    __syncthreads();
    for (int j = t; j < ELASTIC_DRAWS; j += AUG_THREADS) {            // horizontal pass
      const int p = j % AUG_PIX, x = p % 28;
      const int k0 = max(-R, -x), k1 = min(R, 27 - x);
      double acc = 0.0;
      for (int k = k0; k <= k1; ++k) acc = __fma_rn(s_w[abs(k)], (double)s_v[j + k], acc);
      s_h[j] = acc;
    }
    __syncthreads();
    const float4 c = s_coef[r];
    for (int p = t; p < AUG_PIX; p += AUG_THREADS) {                  // vertical pass, then the warp
      const int y = p / 28, x = p - 28 * y;
      const int k0 = max(-R, -y), k1 = min(R, 27 - y);
      float e[2];
#pragma unroll
      for (int d = 0; d < 2; ++d) {
        double acc = 0.0;
        for (int k = k0; k <= k1; ++k) acc = __fma_rn(s_w[abs(k)], s_h[d * AUG_PIX + p + 28 * k], acc);
        e[d] = __double2float_rn(__dmul_rn(ea.alpha, acc));
      }
      if (field_out != nullptr) {
        field_out[(size_t)b * ELASTIC_DRAWS + p] = e[0];
        field_out[(size_t)b * ELASTIC_DRAWS + AUG_PIX + p] = e[1];
      }
      const float dx = __fsub_rn(__fadd_rn((float)x - 13.5f, e[0]), c.z);   // x - 13.5 is exact
      const float dy = __fsub_rn(__fadd_rn((float)y - 13.5f, e[1]), c.w);
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

// As dm_augment_affine, with the elastic field composed in front of the affine map.  alpha: finite, 0 <= alpha <= 64
// (pixels); weights: host memory, the radius + 1 doubles w_0 .. w_radius of augment.gaussian_weights (finite, >= 0), radius
// 0..32.  batch <= floor(2^32 / 1568).  params_out: null, or batch * 8 floats as in dm_augment_affine.  field_out: null,
// or fp32 [batch, 2, 784] receiving the displacement (ex, then ey) each pixel used.  Enqueued on `stream`; advances
// counter[0] by one.
int dm_augment_elastic(const void* src, void* dst, int batch, void* counter, unsigned int seed_mix, double max_shift,
                       double max_rotation, double max_scale, double alpha, const void* weights, int radius,
                       void* params_out, void* field_out, void* stream) {
  using namespace dm;
  if (src == nullptr || dst == nullptr || counter == nullptr || weights == nullptr) return -1;
  if (batch < 1 || batch > ELASTIC_MAX_BATCH || radius < 0 || radius > ELASTIC_MAX_RADIUS) return -1;
  if (!(isfinite(max_shift) && isfinite(max_rotation) && isfinite(max_scale) && isfinite(alpha)) || max_shift < 0.0 ||
      max_rotation < 0.0 || max_scale < 0.0 || max_scale >= 1.0 || alpha < 0.0 || alpha > 64.0)
    return -1;
  ElasticArgs ea{};
  ea.alpha = alpha;
  ea.radius = radius;
  const double* w = reinterpret_cast<const double*>(weights);
  for (int k = 0; k <= radius; ++k) {
    if (!(isfinite(w[k]) && w[k] >= 0.0)) return -1;
    ea.w[k] = w[k];
  }
  const AugRange rg{max_shift, max_rotation, max_scale};
  return (int)launch_kernel(augment_elastic_kernel, dim3(augment_grid(batch, num_sms())), dim3(AUG_THREADS), 0,
                            reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const float*>(src),
                            reinterpret_cast<float*>(dst), batch, reinterpret_cast<unsigned int*>(counter),
                            (uint32_t)seed_mix, rg, ea, reinterpret_cast<float*>(params_out),
                            reinterpret_cast<float*>(field_out));
}

}  // extern "C"
