// Best-scoring weights of the in-training evaluation (--keep_best_checkpoint): the chief's validation pass decides on the
// device whether it scored better than every earlier pass, and if so copies the arena it scored aside.  Both kernels are
// nodes of the pass's graph, after its last eval_head chunk, so keeping the best weights adds no host synchronisation.
//
//   eval_best_decide   1 thread.  A pass improves on the best when it scored the whole validation set (examples == n), its
//                      snapshot -- for a snapshot pass -- was accepted (status > 0), and its correct count is strictly
//                      greater than BestState.correct (ties keep the earlier pass).  It then stores the pass's step, counts
//                      and loss into BestState and sets valid; the decision word gets 1, else 0.  The same test as
//                      eval_target (csrc/eval_target.cu), so a dropped snapshot pass (status -1) never counts.
//   eval_best_copy     grid-stride float4 copy (scalar tail) of the scored fp32 arena -- live arena, snapshot buffer or
//                      moving-average shadow -- into the caller-owned best arena.  Every CTA returns at once when the
//                      decision word is 0.  A separate launch, so every CTA reads the decision decide wrote for this pass.
//
// The copy's loads bypass L1 (ld.global.cg): with the live arena, peers write it over NVLink, and this GPU's L2 is where
// those stores land.  The copy reads nothing but the scored arena, which the pass has just read.
#include "common.cuh"
#include "eval_state.cuh"
#include "host_utils.h"

namespace dm {

constexpr int BEST_THREADS = 512;

// Caller-owned; zeroed once, with `correct` seeded from an earlier run's best (valid stays 0 until a pass improves on it).
struct BestState {
  double loss_sum;             // of the best pass
  uint32_t step;               // global step the best pass scored
  uint32_t correct;            // best count so far (the seed until a pass improves on it)
  uint32_t examples;
  uint32_t valid;              // 1 once a pass of this run became the best: the best arena holds its weights
};

struct BestArgs {
  const EvalState* st;         // the pass's running state, complete once the pass's last chunk has run
  const uint32_t* step_ptr;    // step the pass scored: the epoch word, SnapState.step or the average's step
  const int32_t* status_ptr;   // SnapState.status of a snapshot pass (> 0: accepted), null for any other pass
  uint32_t examples;           // rows of the validation set
  BestState* best;
  uint32_t* decision;          // 1: this pass is the new best, the copy runs
};

__global__ void eval_best_decide_kernel(const __grid_constant__ BestArgs a) {
  if (threadIdx.x != 0) return;
  const EvalState* st = a.st;
  BestState* b = a.best;
  const bool counts = a.status_ptr == nullptr || *a.status_ptr > 0;
  if (!counts || st->examples != a.examples || st->correct <= b->correct) {
    *a.decision = 0u;
    return;
  }
  b->loss_sum = st->loss_sum;
  b->step = *a.step_ptr;
  b->correct = st->correct;
  b->examples = st->examples;
  b->valid = 1u;
  *a.decision = 1u;
}

__global__ void __launch_bounds__(BEST_THREADS) eval_best_copy_kernel(const uint32_t* __restrict__ decision,
                                                                      const float* __restrict__ src,
                                                                      float* __restrict__ dst, long long numel) {
  if (*decision == 0u) return;
  const long long n4 = numel >> 2;
  const long long stride = (long long)gridDim.x * BEST_THREADS;
  for (long long i = (long long)blockIdx.x * BEST_THREADS + threadIdx.x; i < n4; i += stride)
    reinterpret_cast<float4*>(dst)[i] = __ldcg(reinterpret_cast<const float4*>(src) + i);
  // tail: the last numel % 4 elements, one thread each (CTA 0)
  const long long t = 4 * n4 + (long long)blockIdx.x * BEST_THREADS + threadIdx.x;
  if (t < numel) dst[t] = __ldcg(src + t);
}

}  // namespace dm

extern "C" {

int dm_best_state_bytes() { return (int)sizeof(dm::BestState); }

// state: the pass's EvalState (csrc/eval_head.cu); step_ptr: u32 device word; status_ptr: i32 device word or null;
// best: BestState; decision: u32 device word.
int dm_eval_best_decide(const void* state, const void* step_ptr, const void* status_ptr, unsigned int examples, void* best,
                        void* decision, void* stream) {
  if (state == nullptr || step_ptr == nullptr || best == nullptr || decision == nullptr || examples < 1) return -1;
  dm::BestArgs a;
  a.st = reinterpret_cast<const dm::EvalState*>(state);
  a.step_ptr = reinterpret_cast<const uint32_t*>(step_ptr);
  a.status_ptr = reinterpret_cast<const int32_t*>(status_ptr);
  a.examples = examples;
  a.best = reinterpret_cast<dm::BestState*>(best);
  a.decision = reinterpret_cast<uint32_t*>(decision);
  dm::eval_best_decide_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  return (int)cudaGetLastError();
}

// decision: u32 device word (0: nothing is copied); src, dst: fp32 arenas of `numel` floats, 16-byte aligned.
int dm_eval_best_copy(const void* decision, const void* src, void* dst, long long numel, void* stream) {
  if (decision == nullptr || src == nullptr || dst == nullptr || numel < 1 ||
      ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15))
    return -1;
  const long long blocks = (numel / 4 + dm::BEST_THREADS - 1) / dm::BEST_THREADS;
  const int grid = blocks < 1 ? 1 : (blocks < dm::num_sms() ? (int)blocks : dm::num_sms());
  dm::eval_best_copy_kernel<<<grid, dm::BEST_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const uint32_t*>(decision), reinterpret_cast<const float*>(src), reinterpret_cast<float*>(dst),
      numel);
  return (int)cudaGetLastError();
}

}  // extern "C"
