// Host-side helpers shared by the launchers: error macro, driver entry points fetched at
// run time (so the library has no link-time dependency on libcuda and loads on a CPU-only
// box for the build check), TMA tensor-map encoders.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define DM_CUDA_OK(expr)                                                                      \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      fprintf(stderr, "[dmnist] CUDA error %d (%s) at %s:%d: %s\n", (int)_e,                  \
              cudaGetErrorString(_e), __FILE__, __LINE__, #expr);                             \
      return (int)_e;                                                                         \
    }                                                                                         \
  } while (0)

namespace dm {

// Programmatic dependent launch (PDL): every kernel of the training step is launched with the
// programmatic-stream-serialization attribute and executes `griddepcontrol.wait` after its private
// prologue (barrier init, descriptor prefetch), so the next kernel's CTAs are resident and
// set up while the previous kernel drains -- the launch gap between the step's 11 dependent
// kernels disappears (also inside a captured CUDA graph: the edges become programmatic).
extern int g_pdl;
// Upper bound for the persistent kernels' grids (0 = one CTA per SM).  The bucketed aggregation lowers it
// for the backward kernels that run next to the early sync kernel, so those leave SMs free for it.
extern int g_max_ctas;

// Number of SMs of the current device (queried once per process).
int num_sms();
// Grid bound of the persistent kernels: g_max_ctas if set, else num_sms().
inline int max_ctas() { return g_max_ctas > 0 ? g_max_ctas : num_sms(); }

template <typename Kern, typename... Args>
inline cudaError_t launch_kernel(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = g_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

// Resolve a driver API symbol through the runtime (cudaGetDriverEntryPoint).
void* driver_symbol(const char* name);

// 2-D bf16 tensor map.  inner = contiguous dimension (elements), outer = rows,
// ld_elems = elements between rows.  swizzle_bytes in {0, 32, 64, 128}.
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                      uint32_t box_inner, uint32_t box_outer, int swizzle_bytes);

// 4-D bf16 tensor map over an NHWC activation tensor viewed as (C, W, H, N).
int make_tmap_nhwc_bf16(CUtensorMap* out, const void* base, int C, int W, int H, int N, uint32_t box_c,
                        uint32_t box_w, uint32_t box_h, int swizzle_bytes);

// The largest batch a LeNet kernel with a workspace sized at compile time accepts; dm_lenet_max_batch is their minimum.
int fc1_dgrad_unpool_max_batch();   // gemm_tc.cu
int fc2_fwd_bwd_max_batch();        // lenet_simt.cu

// Rows `idx[0..batch)` of a device-resident training set (fp32 images [N, 784], int64 labels [N]) -> an input slot in
// pack_batch's layout (csrc/batch_gather.cu).
cudaError_t launch_gather_batch(const int32_t* idx, const float* images, const int64_t* labels, int batch, void* slot,
                                cudaStream_t stream);

}  // namespace dm
