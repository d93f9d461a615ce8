// Device-resident running state of one in-training validation pass: written by csrc/eval_head.cu, read after the pass by
// the target test of csrc/eval_target.cu.
#pragma once

namespace dm {

// Caller-owned, zero-initialised once.
struct EvalState {
  double loss_sum;                 // sum of per-row cross entropies, chunk after chunk
  unsigned long long t_begin;      // %globaltimer at the start of the pass
  unsigned int correct;
  unsigned int examples;
  unsigned int ticket;             // arrive_last_cta ticket of the chunk in flight
  unsigned int seq;                // records published so far
};

}  // namespace dm
