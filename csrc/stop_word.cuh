// The run's stop step in the replicas' symmetric stop words (csrc/eval_target.cu): shared by every evaluation-pass node that
// can end a run, so a stop step is set once, by whichever decides first.
#pragma once

#include <stdint.h>

namespace dm {

// One thread.  Stores S = `s` into every replica's stop word over NVLink unless this replica's own word is already set (an
// earlier pass, or an earlier node of the same pass, set the stop: it stands), then fence.sc.sys.  True if it stored.
__device__ __forceinline__ bool store_stop_once(uint32_t* const* stop, int rank, int nranks, uint32_t s) {
  if (*reinterpret_cast<volatile uint32_t*>(stop[rank]) != 0u) return false;
  for (int r = 0; r < nranks; ++r) *reinterpret_cast<volatile uint32_t*>(stop[r]) = s;
  // orders the stores before everything the chief's stream does after this kernel, in particular before its next step's
  // exchange, which every peer has to observe before it can finish that step
  __threadfence_system();
  return true;
}

}  // namespace dm
