// Device-resident training set: gather one step's batch from a table that lives in GPU memory.
//
// With the training set uploaded once (fp32 images [N, 784], int64 labels [N]), a step's input is B int32 row indices
// instead of the B * 3144-byte packed batch.  gather_batch_kernel copies the indexed rows into an input slot in exactly the
// layout pack_batch / load_packed produce -- fp32 images [B, 784], then int64 labels [B] -- so the step graphs read the
// same bytes whichever way the slot was filled.  It runs on the engine's copy stream, where the batch DMA runs otherwise.
//
// One thread per 16-byte piece: a row is 196 float4 and the slot's label block starts at B * 3136 bytes, so every image
// access is a 16-byte load / store on a 16-byte boundary; the first B threads also copy one label each.  The indices are
// checked on the host to lie in [0, N) before anything is enqueued.
#include <stdint.h>

#include "host_utils.h"

namespace dm {

constexpr int GATHER_THREADS = 256;
constexpr int ROW_VEC = 784 / 4;          // float4 per image row

__global__ void __launch_bounds__(GATHER_THREADS) gather_batch_kernel(const int32_t* __restrict__ idx,
                                                                       const float4* __restrict__ images,
                                                                       const int64_t* __restrict__ labels, int batch,
                                                                       float4* __restrict__ slot_images,
                                                                       int64_t* __restrict__ slot_labels) {
  const int t = blockIdx.x * GATHER_THREADS + threadIdx.x;
  if (t >= batch * ROW_VEC) return;
  const int b = t / ROW_VEC;
  const int c = t - b * ROW_VEC;
  const int64_t row = __ldg(idx + b);
  slot_images[t] = __ldg(images + row * ROW_VEC + c);
  if (t < batch) slot_labels[t] = __ldg(labels + __ldg(idx + t));
}

// The slot's images at `slot`, its labels right behind them (pack_batch's layout).
cudaError_t launch_gather_batch(const int32_t* idx, const float* images, const int64_t* labels, int batch, void* slot,
                                cudaStream_t stream) {
  if (batch <= 0) return cudaErrorInvalidValue;
  float4* out = reinterpret_cast<float4*>(slot);
  int64_t* out_labels = reinterpret_cast<int64_t*>(out + (size_t)batch * ROW_VEC);
  const int blocks = (batch * ROW_VEC + GATHER_THREADS - 1) / GATHER_THREADS;
  gather_batch_kernel<<<blocks, GATHER_THREADS, 0, stream>>>(idx, reinterpret_cast<const float4*>(images), labels, batch,
                                                             out, out_labels);
  return cudaGetLastError();
}

}  // namespace dm

extern "C" {

// idx: `batch` int32 row indices (device memory, each in [0, rows of the table)); images: fp32 [N, 784], labels: int64 [N]
// (device memory, 16-byte aligned); slot: batch * 3144 bytes of device memory.  Enqueued on `stream`.
int dm_gather_batch(const void* idx, const void* images, const void* labels, int batch, void* slot, void* stream) {
  DM_CUDA_OK(dm::launch_gather_batch(reinterpret_cast<const int32_t*>(idx), reinterpret_cast<const float*>(images),
                                     reinterpret_cast<const int64_t*>(labels), batch, slot,
                                     reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

}  // extern "C"
