// Native step executor: the per-step host work of the training loop -- wait for the input slot, DMA the packed batch, chain
// the events, launch the step's CUDA graph, record completion -- as ONE C call instead of ~8 Python-dispatched torch calls
// (interpreter time per step comparable to the step itself).  The reference's equivalent layer is the TF
// session runtime driving `sess.run(train_op, feed_dict)` (src/distributed_train.py:309-335); here the device work is a
// pre-instantiated cudaGraphExec_t per input slot and the host's job is six driver calls.
#include <stdint.h>

#include "host_utils.h"

namespace dm {

struct StepRunner {
  cudaStream_t compute, copy;
  cudaGraphExec_t graph[2];
  void* slot_dev[2];
  size_t in_bytes;
  cudaEvent_t copy_done[2], slot_free[2];
  unsigned long long launched;
  // device-resident training set (dm_runner_arm_gather): per-slot device index buffers and the table
  void* idx_dev[2];
  const float* table_images;
  const int64_t* table_labels;
  int batch;
};

}  // namespace dm

extern "C" {

// graphs: one instantiated graph per input slot (torch.cuda.CUDAGraph.raw_cuda_graph_exec()); slots: the device input buffers
// the graphs read; first_slot: slot of the next step (continues the engine's alternation).
void* dm_runner_create(void* compute_stream, void* copy_stream, void* graph0, void* graph1, void* slot0, void* slot1,
                       unsigned long long in_bytes, int first_slot) {
  using namespace dm;
  StepRunner* r = new StepRunner();
  r->compute = reinterpret_cast<cudaStream_t>(compute_stream);
  r->copy = reinterpret_cast<cudaStream_t>(copy_stream);
  r->graph[0] = reinterpret_cast<cudaGraphExec_t>(graph0);
  r->graph[1] = reinterpret_cast<cudaGraphExec_t>(graph1);
  r->slot_dev[0] = slot0;
  r->slot_dev[1] = slot1;
  r->in_bytes = in_bytes;
  r->launched = (unsigned long long)(first_slot & 1);
  for (int i = 0; i < 2; ++i) {
    if (cudaEventCreateWithFlags(&r->copy_done[i], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&r->slot_free[i], cudaEventDisableTiming) != cudaSuccess) {
      delete r;
      return nullptr;
    }
  }
  return r;
}

// One training step: packed batch `src` (page-locked host memory or device memory, in_bytes long) -> slot -> graph.
// Returns the slot used (0 / 1) or a negative CUDA error code.
int dm_runner_step(void* h, const void* src) {
  using namespace dm;
  StepRunner* r = reinterpret_cast<StepRunner*>(h);
  const int s = (int)(r->launched & 1ull);
  cudaError_t e;
  if ((e = cudaStreamWaitEvent(r->copy, r->slot_free[s], 0)) != cudaSuccess) return -(int)e;     // the step that last read the slot is done
  if ((e = cudaMemcpyAsync(r->slot_dev[s], src, r->in_bytes, cudaMemcpyDefault, r->copy)) != cudaSuccess) return -(int)e;
  if ((e = cudaEventRecord(r->copy_done[s], r->copy)) != cudaSuccess) return -(int)e;
  if ((e = cudaStreamWaitEvent(r->compute, r->copy_done[s], 0)) != cudaSuccess) return -(int)e;
  if ((e = cudaGraphLaunch(r->graph[s], r->compute)) != cudaSuccess) return -(int)e;
  if ((e = cudaEventRecord(r->slot_free[s], r->compute)) != cudaSuccess) return -(int)e;
  r->launched += 1;
  return s;
}

// Device-resident training set for dm_runner_step_indices: idx0 / idx1 are the slots' device index buffers (batch int32
// each), images / labels the table (fp32 [N, 784], int64 [N]).
int dm_runner_arm_gather(void* h, void* idx0, void* idx1, const void* images, const void* labels, int batch) {
  dm::StepRunner* r = reinterpret_cast<dm::StepRunner*>(h);
  r->idx_dev[0] = idx0;
  r->idx_dev[1] = idx1;
  r->table_images = reinterpret_cast<const float*>(images);
  r->table_labels = reinterpret_cast<const int64_t*>(labels);
  r->batch = batch;
  return 0;
}

// One training step from `batch` row indices of the armed table (page-locked host memory, each in [0, N)): the same event
// chain as dm_runner_step, with the batch DMA replaced by an index DMA plus the gather kernel on the copy stream.
// Returns the slot used (0 / 1) or a negative CUDA error code.
int dm_runner_step_indices(void* h, const void* idx_host) {
  using namespace dm;
  StepRunner* r = reinterpret_cast<StepRunner*>(h);
  if (r->table_images == nullptr) return -(int)cudaErrorInvalidValue;
  const int s = (int)(r->launched & 1ull);
  cudaError_t e;
  if ((e = cudaStreamWaitEvent(r->copy, r->slot_free[s], 0)) != cudaSuccess) return -(int)e;
  if ((e = cudaMemcpyAsync(r->idx_dev[s], idx_host, (size_t)r->batch * sizeof(int32_t), cudaMemcpyHostToDevice, r->copy)) !=
      cudaSuccess)
    return -(int)e;
  if ((e = launch_gather_batch(reinterpret_cast<const int32_t*>(r->idx_dev[s]), r->table_images, r->table_labels, r->batch,
                               r->slot_dev[s], r->copy)) != cudaSuccess)
    return -(int)e;
  if ((e = cudaEventRecord(r->copy_done[s], r->copy)) != cudaSuccess) return -(int)e;
  if ((e = cudaStreamWaitEvent(r->compute, r->copy_done[s], 0)) != cudaSuccess) return -(int)e;
  if ((e = cudaGraphLaunch(r->graph[s], r->compute)) != cudaSuccess) return -(int)e;
  if ((e = cudaEventRecord(r->slot_free[s], r->compute)) != cudaSuccess) return -(int)e;
  r->launched += 1;
  return s;
}

// Block the calling host thread until the step that last used `slot` has completed (its results are in host memory).
int dm_runner_wait(void* h, int slot) {
  dm::StepRunner* r = reinterpret_cast<dm::StepRunner*>(h);
  return (int)cudaEventSynchronize(r->slot_free[slot & 1]);
}

// Block the calling host thread until the input DMA (and gather) last enqueued for `slot` has completed: its host source
// may then be rewritten or freed.
int dm_runner_wait_copy(void* h, int slot) {
  dm::StepRunner* r = reinterpret_cast<dm::StepRunner*>(h);
  return (int)cudaEventSynchronize(r->copy_done[slot & 1]);
}

// 1: that step has completed, 0: still running, < 0: error.
int dm_runner_query(void* h, int slot) {
  dm::StepRunner* r = reinterpret_cast<dm::StepRunner*>(h);
  cudaError_t e = cudaEventQuery(r->slot_free[slot & 1]);
  if (e == cudaSuccess) return 1;
  if (e == cudaErrorNotReady) return 0;
  return -(int)e;
}

void dm_runner_destroy(void* h) {
  dm::StepRunner* r = reinterpret_cast<dm::StepRunner*>(h);
  if (r == nullptr) return;
  for (int i = 0; i < 2; ++i) {
    cudaEventDestroy(r->copy_done[i]);
    cudaEventDestroy(r->slot_free[i]);
  }
  delete r;
}

}  // extern "C"
