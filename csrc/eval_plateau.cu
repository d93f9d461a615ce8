// Learning-rate cuts at a plateau (--lr_plateau_patience): the chief's in-training validation pass decides on the device
// whether the run has stopped improving, and if so schedules a cut of the learning rate in every replica's cut table.
//
//   eval_plateau       1 thread, the last node of the pass's graph (after eval_best_*, eval_target and eval_patience).  A
//                      pass counts when it scored the whole validation set (examples == n) and, for a snapshot pass, its
//                      snapshot was accepted (status > 0): the test of eval_patience.  The first counting pass sets the
//                      baseline (best = correct, since = 0); after it, a counting pass with correct > best + min_delta
//                      rows sets best = correct and since = 0, any other counting pass increments since.  When since
//                      reaches the patience P, the pass's step g triggers a cut: since = 0, best is kept, and unless
//                      SYNC_MAX_CUTS cuts are already scheduled, S = g + margin goes into entry `cuts` of every replica's
//                      cut table and cuts += 1.  A pass that does not count changes nothing.
//
// The cut tables are one symmetric allocation (FusedBackend.allocate_buffer), SYNC_MAX_CUTS u32 per replica, 0xFFFFFFFF
// until a cut is stored there.  Only the chief writes them, each entry at most once, so a reader sees either no cut or the
// final step of that cut.  The aggregation kernels read their own replica's table in cta_scale (fused_sync.cuh).  Why every
// replica of a K = N run applies cut k from the same step S_k: DESIGN §4 (learning-rate cuts), which rests on §4.4.
//
// The host rule it mirrors is lr_plateau.advance; the training loop replays it over the pass records for its report.
#include <stdint.h>

#include "eval_state.cuh"
#include "fused_sync.cuh"

namespace dm {

// Caller-owned; zeroed once per run, with `cuts` seeded from the cuts a restarted run keeps.
struct PlateauState {
  uint32_t best;               // correct count to beat (by more than min_delta rows)
  uint32_t since;              // counting passes since the best or the last trigger
  uint32_t baseline;           // 1 once a counting pass set best
  uint32_t cuts;               // cuts scheduled so far (entries 0 .. cuts-1 of every table are set)
  uint32_t trigger_step;       // global step of the last pass that triggered a cut (0 until one did)
};

struct PlateauArgs {
  const EvalState* st;          // the pass's running state, complete once the pass's last chunk has run
  const uint32_t* step_ptr;     // step the pass scored: the epoch word, SnapState.step or the average's step
  const int32_t* status_ptr;    // SnapState.status of a snapshot pass (> 0: accepted), null for any other pass
  uint32_t examples;            // rows of the validation set
  uint32_t patience;            // P >= 1
  uint32_t min_delta;           // rows a pass must beat the best by
  uint32_t margin;              // S = step + margin
  PlateauState* ps;
  int nranks;
  uint32_t* tables[SYNC_MAX_RANKS];   // every replica's cut table
};

__global__ void eval_plateau_kernel(const __grid_constant__ PlateauArgs a) {
  if (threadIdx.x != 0) return;
  if (a.status_ptr != nullptr && *a.status_ptr <= 0) return;
  const EvalState* st = a.st;
  if (st->examples != a.examples) return;
  PlateauState* p = a.ps;
  const uint32_t step = *a.step_ptr, correct = st->correct;
  if (p->baseline == 0u || (uint64_t)correct > (uint64_t)p->best + a.min_delta) {
    p->best = correct;
    p->since = 0u;
    p->baseline = 1u;
    return;
  }
  if (++p->since < a.patience) return;
  p->since = 0u;
  p->trigger_step = step;
  const uint32_t k = p->cuts;
  if (k >= (uint32_t)SYNC_MAX_CUTS) return;                                  // over the cap: the trigger is ignored
  const uint32_t s = step + a.margin;
  for (int r = 0; r < a.nranks; ++r) *reinterpret_cast<volatile uint32_t*>(a.tables[r] + k) = s;
  p->cuts = k + 1u;
  // orders the stores before everything the chief's stream does after this kernel, in particular before its next step's
  // exchange, which every peer has to observe before it can finish that step
  __threadfence_system();
}

}  // namespace dm

extern "C" {

int dm_plateau_state_bytes() { return (int)sizeof(dm::PlateauState); }

// state: the pass's EvalState (csrc/eval_head.cu); step_ptr: u32 device word; status_ptr: i32 device word or null;
// plateau_state: PlateauState; tables: table of `nranks` device pointers to the replicas' cut tables (index = rank).
int dm_eval_plateau(const void* state, const void* step_ptr, const void* status_ptr, unsigned int examples,
                    unsigned int patience, unsigned int min_delta, unsigned int margin, void* plateau_state,
                    void* const* tables, int nranks, void* stream) {
  if (state == nullptr || step_ptr == nullptr || plateau_state == nullptr || tables == nullptr || examples < 1 ||
      patience < 1 || min_delta >= examples || margin < 1 || nranks < 1 || nranks > dm::SYNC_MAX_RANKS)
    return -1;
  dm::PlateauArgs a;
  a.st = reinterpret_cast<const dm::EvalState*>(state);
  a.step_ptr = reinterpret_cast<const uint32_t*>(step_ptr);
  a.status_ptr = reinterpret_cast<const int32_t*>(status_ptr);
  a.examples = examples;
  a.patience = patience;
  a.min_delta = min_delta;
  a.margin = margin;
  a.ps = reinterpret_cast<dm::PlateauState*>(plateau_state);
  a.nranks = nranks;
  for (int r = 0; r < dm::SYNC_MAX_RANKS; ++r) a.tables[r] = r < nranks ? reinterpret_cast<uint32_t*>(tables[r]) : nullptr;
  dm::eval_plateau_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  return (int)cudaGetLastError();
}

}  // extern "C"
