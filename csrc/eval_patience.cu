// Early stopping with a patience (--early_stopping_patience): the chief's in-training validation pass decides on the device
// whether the run has stopped improving, and sets the stop step the way --target_accuracy does (csrc/eval_target.cu).
//
//   eval_patience      1 thread, the last node of the pass's graph (after eval_best_* and eval_target).  A pass counts when
//                      it scored the whole validation set (examples == n) and, for a snapshot pass, its snapshot was
//                      accepted (status > 0): the test of eval_best_decide and eval_target.  The first counting pass sets
//                      the baseline (best = correct, since = 0); after it, a counting pass with correct > best + min_delta
//                      rows sets best = correct and since = 0, any other counting pass increments since.  A pass that does
//                      not count changes nothing.  When since reaches the patience P, the pass's step g is the trigger
//                      step and S = g + margin goes into every replica's stop word unless a stop is already set
//                      (store_stop_once, stop_word.cuh).  From then on the state is frozen.
//
// The host rule it mirrors is early_stopping.advance; the training loop replays it over the pass records for its report.
#include <stdint.h>

#include "eval_state.cuh"
#include "fused_sync.cuh"
#include "stop_word.cuh"

namespace dm {

// Caller-owned, zeroed once per run.
struct PatienceState {
  uint32_t best;               // correct count to beat (by more than min_delta rows)
  uint32_t since;              // counting passes since the best; == patience once exhausted
  uint32_t best_step;          // global step the best pass scored
  uint32_t trigger_step;       // global step of the pass that exhausted the patience (valid once since == patience)
  uint32_t baseline;           // 1 once a counting pass set best
};

struct PatienceArgs {
  const EvalState* st;          // the pass's running state, complete once the pass's last chunk has run
  const uint32_t* step_ptr;     // step the pass scored: the epoch word, SnapState.step or the average's step
  const int32_t* status_ptr;    // SnapState.status of a snapshot pass (> 0: accepted), null for any other pass
  uint32_t examples;            // rows of the validation set
  uint32_t patience;            // P >= 1
  uint32_t min_delta;           // rows a pass must beat the best by
  uint32_t margin;              // S = step + margin
  PatienceState* ps;
  int rank, nranks;
  uint32_t* stop[SYNC_MAX_RANKS];   // every replica's stop word
};

__global__ void eval_patience_kernel(const __grid_constant__ PatienceArgs a) {
  if (threadIdx.x != 0) return;
  PatienceState* p = a.ps;
  if (p->since >= a.patience) return;                                       // exhausted by an earlier pass
  if (a.status_ptr != nullptr && *a.status_ptr <= 0) return;
  const EvalState* st = a.st;
  if (st->examples != a.examples) return;
  const uint32_t step = *a.step_ptr, correct = st->correct;
  if (p->baseline == 0u || (uint64_t)correct > (uint64_t)p->best + a.min_delta) {
    p->best = correct;
    p->best_step = step;
    p->since = 0u;
    p->baseline = 1u;
    return;
  }
  if (++p->since < a.patience) return;
  p->trigger_step = step;
  store_stop_once(a.stop, a.rank, a.nranks, step + a.margin);
}

}  // namespace dm

extern "C" {

int dm_patience_state_bytes() { return (int)sizeof(dm::PatienceState); }

// state: the pass's EvalState (csrc/eval_head.cu); step_ptr: u32 device word; status_ptr: i32 device word or null;
// patience_state: PatienceState; stop: table of `nranks` device pointers to the replicas' u32 stop words (index = rank).
int dm_eval_patience(const void* state, const void* step_ptr, const void* status_ptr, unsigned int examples,
                     unsigned int patience, unsigned int min_delta, unsigned int margin, void* patience_state,
                     void* const* stop, int rank, int nranks, void* stream) {
  if (state == nullptr || step_ptr == nullptr || patience_state == nullptr || stop == nullptr || examples < 1 ||
      patience < 1 || min_delta >= examples || margin < 1 || nranks < 1 || nranks > dm::SYNC_MAX_RANKS || rank < 0 ||
      rank >= nranks)
    return -1;
  dm::PatienceArgs a;
  a.st = reinterpret_cast<const dm::EvalState*>(state);
  a.step_ptr = reinterpret_cast<const uint32_t*>(step_ptr);
  a.status_ptr = reinterpret_cast<const int32_t*>(status_ptr);
  a.examples = examples;
  a.patience = patience;
  a.min_delta = min_delta;
  a.margin = margin;
  a.ps = reinterpret_cast<dm::PatienceState*>(patience_state);
  a.rank = rank;
  a.nranks = nranks;
  for (int r = 0; r < dm::SYNC_MAX_RANKS; ++r) a.stop[r] = r < nranks ? reinterpret_cast<uint32_t*>(stop[r]) : nullptr;
  dm::eval_patience_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  return (int)cudaGetLastError();
}

}  // extern "C"
