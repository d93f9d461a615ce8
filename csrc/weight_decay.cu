// Loss term of the L2 weight decay (--weight_decay): the step's loss word gains (float)(lambda * R), R = sum of v^2 / 2 over
// the decayed variables.  The weight-gradient kernels that add lambda * v to those variables' gradients also store the
// sum of the squares they read, one double per CTA (dm_gemm_bf16_decay, dm_fc2_wgrad_decay); this kernel adds the
// partials in index order, in double, so two runs on the same weights produce the same loss word.
//
//   weight_decay_loss   one warp: lane l sums partials l, l + 32, ... in order, then a fixed butterfly.  Stores R into
//                       part[n] and adds (float)(lambda * R) to loss_acc[0].
#include "common.cuh"
#include "host_utils.h"

namespace dm {

__global__ void __launch_bounds__(32) weight_decay_loss_kernel(double* part, int n, float decay, float* loss_acc) {
  pdl_wait();
  const int lane = threadIdx.x;
  double s = 0.0;
  for (int i = lane; i < n; i += 32) s += part[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const double r = 0.5 * s;
    part[n] = r;
    loss_acc[0] += __double2float_rn((double)decay * r);
  }
}

}  // namespace dm

extern "C" {

// part: n + 1 doubles (the n partials, then R); loss_acc: the step's (loss, accuracy) words.
int dm_weight_decay_loss(void* part, int n, float decay, void* loss_acc, void* stream) {
  if (part == nullptr || loss_acc == nullptr || n < 1) return -1;
  return (int)dm::launch_kernel(dm::weight_decay_loss_kernel, dim3(1), dim3(32), 0, reinterpret_cast<cudaStream_t>(stream),
                                reinterpret_cast<double*>(part), n, decay, reinterpret_cast<float*>(loss_acc));
}

}  // extern "C"
