// Quality-target stop of a training run (--target_accuracy): the chief's in-training validation pass decides on the device
// whether the run has reached its target, and every replica learns the stop step at the end of its own steps.
//
//   tta_stamp          1 thread: %globaltimer at the start of the run's first step (t0 of the reported training time)
//   eval_target        1 thread, right after an evaluation pass on the chief's training stream (inside the pass's graph):
//                      a complete pass with correct >= need -- and, for a snapshot pass, an accepted snapshot -- that finds
//                      no stop set yet stores S = (step the pass scored) + margin into every replica's stop word over NVLink,
//                      then fence.sc.sys.  A dropped snapshot pass (status -1) never counts.
//   stop_publish       1 thread, the last node of every replica's step graph: acquire load of the replica's own stop word,
//                      stored into a page-locked host word that the host reads after the step's completion event.
//
// The stop words are one symmetric allocation (FusedBackend.allocate_buffer), 0 until a stop is set; only the chief writes
// them, once (store_stop_once, stop_word.cuh: eval_patience, csrc/eval_patience.cu, may set the stop instead).  Why every replica of a K = N run stops at the same S, and why margin = 2: DESIGN §4.4.
#include <stdint.h>

#include "eval_state.cuh"
#include "fused_sync.cuh"
#include "stop_word.cuh"

namespace dm {

struct TargetArgs {
  const EvalState* st;          // the pass's running state, complete once the pass's last chunk has run
  const uint32_t* step_ptr;     // step the pass scored: the epoch word (live pass) or SnapState.step
  const int32_t* status_ptr;    // SnapState.status of a snapshot pass (> 0: accepted), null for a live pass
  uint32_t need;                // smallest correct count that reaches the target
  uint32_t examples;            // rows of the validation set: a pass that scored fewer is not a pass over the set
  uint32_t margin;              // S = step + margin
  int rank, nranks;
  uint32_t* stop[SYNC_MAX_RANKS];   // every replica's stop word
};

__global__ void tta_stamp_kernel(unsigned long long* t) { *t = globaltimer_ns(); }

__global__ void eval_target_kernel(const __grid_constant__ TargetArgs a) {
  if (threadIdx.x != 0) return;
  if (a.status_ptr != nullptr && *a.status_ptr <= 0) return;
  const EvalState* st = a.st;
  if (st->examples != a.examples || st->correct < a.need) return;
  store_stop_once(a.stop, a.rank, a.nranks, *a.step_ptr + a.margin);
}

__global__ void stop_publish_kernel(const uint32_t* stop, volatile uint32_t* host) {
  *host = ld_acquire_sys(stop);
}

}  // namespace dm

extern "C" {

int dm_tta_stamp(void* t_ns, void* stream) {
  dm::tta_stamp_kernel<<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<unsigned long long*>(t_ns));
  return (int)cudaGetLastError();
}

// state: the pass's EvalState (csrc/eval_head.cu); step_ptr: u32 device word; status_ptr: i32 device word or null;
// stop: table of `nranks` device pointers to the replicas' u32 stop words (index = rank).
int dm_eval_target(const void* state, const void* step_ptr, const void* status_ptr, unsigned int need,
                   unsigned int examples, unsigned int margin, void* const* stop, int rank, int nranks, void* stream) {
  if (nranks < 1 || nranks > dm::SYNC_MAX_RANKS || rank < 0 || rank >= nranks || need < 1 || need > examples ||
      margin < 1)
    return -1;
  dm::TargetArgs a;
  a.st = reinterpret_cast<const dm::EvalState*>(state);
  a.step_ptr = reinterpret_cast<const uint32_t*>(step_ptr);
  a.status_ptr = reinterpret_cast<const int32_t*>(status_ptr);
  a.need = need;
  a.examples = examples;
  a.margin = margin;
  a.rank = rank;
  a.nranks = nranks;
  for (int r = 0; r < dm::SYNC_MAX_RANKS; ++r) a.stop[r] = r < nranks ? reinterpret_cast<uint32_t*>(stop[r]) : nullptr;
  dm::eval_target_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  return (int)cudaGetLastError();
}

// stop: this replica's u32 stop word; host_word: page-locked host memory.
int dm_stop_publish(const void* stop, void* host_word, void* stream) {
  dm::stop_publish_kernel<<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint32_t*>(stop), reinterpret_cast<volatile uint32_t*>(host_word));
  return (int)cudaGetLastError();
}

}  // extern "C"
