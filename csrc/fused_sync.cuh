// Shared definitions of the gradient-aggregation kernels (csrc/fused_sync.cu: single-kernel K-of-N / interval path;
// csrc/fused_bucket.cu: bucketed, overlapped K == N path): the symmetric control block, the peer pointer tables and the
// system-scope memory / multimem helpers.
#pragma once

#include <stddef.h>
#include <string.h>

#include "common.cuh"
#include "host_utils.h"

namespace dm {

constexpr int SYNC_MAX_RANKS = 8;
constexpr int SYNC_RING = 64;          // commit-word ring (steps)
constexpr int SYNC_THREADS = 512;
constexpr int TIMING_RING = 1024;      // per-rank arrival-timestamp ring (steps)
constexpr int SYNC_MAX_CUTS = 32;      // learning-rate cuts per run (SyncCtrl::lr_cuts, lr_plateau.MAX_CUTS)

// Control block, one per rank, in symmetric memory.  Words written remotely are spread over
// separate 128-byte lines.
struct SyncCtrl {
  // ---- written by peers -----------------------------------------------------------------
  volatile uint32_t arrive[SYNC_MAX_RANKS * 32];     // [p*32]: peer p arrived for epoch (value = epoch+1)
  volatile uint32_t done[SYNC_MAX_RANKS * 32];       // [p*32]: peer p's pushes for step s landed (value = s+1)
  volatile unsigned long long commit_local[SYNC_RING];  // ((step+1) << 32) | mask, broadcast by the committer
  // ---- authoritative on the chief only ------------------------------------------------------
  unsigned int bitmap[SYNC_RING];                    // arrival bitmap of step s at [s % RING]
  unsigned long long commit[SYNC_RING];              // ((step+1) << 32) | mask
  volatile uint32_t global_step;                     // number of committed steps
  volatile uint32_t last_in_mask[SYNC_MAX_RANKS];    // (last step in whose mask rank q was) + 1
  uint32_t pad0[32];
  // ---- local ----------------------------------------------------------------------------------
  uint32_t epoch;                // global step of my weights (device-resident so CUDA graphs replay)
  uint32_t cta_counter;          // grid-wide completion counter
  volatile uint32_t decided_tag; // epoch+1 once `decided_mask` is valid for this launch
  volatile uint32_t decided_mask;
  volatile uint32_t decided_late;   // 1: my gradient is not part of the mean
  volatile uint32_t decided_target; // epoch to move to after this launch
  uint32_t error;                // watchdog: 1 = arrival timeout, 2 = done timeout
  uint32_t accepted_steps, dropped_steps;
  uint32_t last_mask, last_count, last_late;
  uint32_t pad1[23];
  // learning-rate schedule (--lr_warmup_steps, --lr_cosine_decay_steps): linear warmup over the first W global steps from
  // the factor f0, and TF's cosine_decay over T steps with the floor alpha in place of the staircase decay; W = T = 0: off.
  // Set once by dm_sync_set_lr_schedule, read by cta_scale.  These words were padding, like the cut table's below.
  uint32_t lr_warmup_steps;      // W
  uint32_t lr_cosine_steps;      // T
  double lr_warmup_start;        // f0
  double lr_cosine_alpha;        // alpha
  // learning-rate cuts (--lr_plateau_patience, csrc/eval_plateau.cu): this replica's table of SYNC_MAX_CUTS cut steps
  // (0xFFFFFFFF = no cut), written by the chief's eval_plateau over NVLink; null when no table is armed.  Set once by
  // dm_sync_set_lr_cuts.  These words were padding: the size and every other offset of the block are unchanged.
  const uint32_t* lr_cuts;
  double lr_factor;              // F: the rate is multiplied by F^c, c = cuts in effect
  unsigned long long t_arrive[TIMING_RING];   // %globaltimer at arrival, per local step (cdf telemetry)
  unsigned long long t_start[TIMING_RING];    // %globaltimer stamped by the step's first kernel
  unsigned long long t_phase[8];              // last launch: kernel start, decided, reduced, pushed, landed, shadowed
  // ---- bucketed (overlapped) aggregation: the early bucket has its own handshake words ---------------------------
  volatile uint32_t arrive_e[SYNC_MAX_RANKS * 32];   // [p*32]: peer p's early-bucket gradients are complete (epoch+1)
  volatile uint32_t done_e[SYNC_MAX_RANKS * 32];     // [p*32]: peer p's early-bucket pushes have landed (epoch+1)
  uint32_t cta_counter_e;
  uint32_t cta_counter2;         // late bucket kernel: CTAs that have finished (the last one closes the step)
  uint32_t pad2[30];
  unsigned long long t_phase_e[8];            // early kernel: start, arrived, reduced (CTA 0), all pushed, all landed, applied (CTA 0)
  // ---- device-side interval mode (mode C, csrc/fused_interval.cu) ------------------------------------------------------------
  volatile unsigned long long iv_state;    // ((step+1) << 32) | gradients accumulated for that step -- read by the committer
  volatile uint32_t iv_busy;               // step+1 while an accumulate for that step is in flight (Dekker pair of commit_local)
  volatile uint32_t iv_last_total;         // written by the committer: divisor of the tick that produced my current weights
  unsigned long long iv_deadline;          // local %globaltimer deadline of the current tick
  unsigned long long iv_interval_ns;
  uint32_t iv_adopted;                     // this iteration adopted new weights: refresh the bf16 shadow
  uint32_t iv_go;                          // this iteration's gradient may be accumulated (its step is still open)
  uint32_t iv_commit_go;                   // step+1: I won the commit of that step -> the apply kernel reduces + pushes
  uint32_t iv_commit_mask;                 // contributors of the tick I am committing
  uint32_t iv_commit_total;                // its divisor (sum of the contributors' counts)
  uint32_t iv_ticks_committed;             // ticks this rank committed (statistics)
  uint32_t cta_counter_iv;
  // ---- host mirror of the status words: the kernel that closes a step writes (epoch, error, accepted, dropped, last_mask,
  // last_count, last_late, seq) into page-locked HOST memory (zero-copy store over PCIe) so the training loop learns a step's
  // outcome without a device read or a memcpy node in the step graph (a D2H memcpy node adds a copy to the graph) ------------------
  uint32_t status_seq;                     // number of steps closed so far (ring index of the mirror slot = seq & 3)
  uint32_t* host_mirror;                   // 4 slots x 8 words in mapped pinned host memory, or null
  uint32_t decider_claim;                  // step+1 of the newest launch whose arrival/commit decision a CTA has claimed
  uint32_t bar_seq;                        // device barriers completed so far (dm_device_barrier)
  // ---- asynchronous SGD (csrc/fused_async.cu): these words were padding ------------------------------------------------------
  uint32_t as_pull;                        // r: the chief's update counter when this iteration pulled its weights
  uint32_t as_ticket;                      // s: the global step this iteration's update produces
  uint32_t pad3[12];
  volatile uint32_t bar[SYNC_MAX_RANKS * 32];   // [p*32]: peer p entered device barrier number (value)
};
static_assert(SYNC_MAX_CUTS == 32, "cta_scale reads one cut-table entry per lane of a warp");
static_assert(offsetof(SyncCtrl, lr_cuts) % 8 == 0 && offsetof(SyncCtrl, lr_factor) + 8 == offsetof(SyncCtrl, t_arrive),
              "the cut-table words take the place of pad1's last words, with no change to the layout around them");
static_assert(sizeof(SyncCtrl) == 23520 && offsetof(SyncCtrl, pad1) == 3540 && offsetof(SyncCtrl, lr_warmup_steps) == 3632 &&
                  offsetof(SyncCtrl, lr_cuts) == 3656 && offsetof(SyncCtrl, t_arrive) == 3672 &&
                  offsetof(SyncCtrl, bar) == 22496,
              "the schedule words take the place of pad1's last words before the cut table: the size of the block and "
              "every other offset are unchanged");
static_assert(offsetof(SyncCtrl, as_ticket) + 4 == offsetof(SyncCtrl, pad3) && offsetof(SyncCtrl, pad3) + 48 == offsetof(SyncCtrl, bar),
              "the asynchronous-SGD words take the place of pad3's first words, with no change to the layout around them");

struct SyncPeers {
  SyncCtrl* ctrl[SYNC_MAX_RANKS];
  float* params[SYNC_MAX_RANKS];
  const float* grads[SYNC_MAX_RANKS];
};

struct SyncArgs {
  int rank, nranks, k;
  int numel4;                 // arena length in float4
  double lr0, decay_rate;     // staircase exponential decay evaluated on device (reference K12), see cta_scale
  int decay_steps;
  float drop_keep;            // gradient drop-connect keep probability, <= 0: off (reference K14)
  uint32_t drop_seed;
  unsigned long long timeout_ns;
  __nv_bfloat16* shadow;      // local bf16 copy of the parameter arena (tensor-core operand source)
  // NVLS (NVSwitch multicast) views of the two arenas, null when the fabric has none.  A load from mc_grads returns the
  // SUM over all ranks computed inside the switch; a store to mc_params lands in every rank's arena.
  const float* mc_grads;
  float* mc_params;
};

// ---- system-scope memory helpers ----------------------------------------------------------------
DMNIST_DEVICE uint32_t ld_acquire_sys(const volatile uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
DMNIST_DEVICE unsigned long long ld_acquire_sys64(const volatile unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// Polling loads: RELAXED (an acquire load costs a CCTL.IVALL -- it invalidates the SM's whole L1 -- on EVERY poll, which is
// poison for the tensor-core kernels the small aggregation CTAs are co-resident with); the one acquire fence a wait needs is
// issued by spin_until() when the wait is over.
DMNIST_DEVICE uint32_t ld_relaxed_sys(const volatile uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
DMNIST_DEVICE unsigned long long ld_relaxed_sys64(const volatile unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
DMNIST_DEVICE void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
DMNIST_DEVICE void st_release_sys(volatile uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
DMNIST_DEVICE void st_release_sys64(volatile unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
DMNIST_DEVICE float4 ld_peer_f4(const float* p) {   // peer data: read once, keep out of L1
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
DMNIST_DEVICE void st_peer_f4(float* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

// In-switch reduction: one 16-byte load returns the element-wise fp32 sum of the same address on every rank.
DMNIST_DEVICE float4 multimem_ld_reduce_f4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
// Multicast store: the switch replicates the 16 bytes into every rank's copy.
DMNIST_DEVICE void multimem_st_f4(float* mc, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

// Host mirror of a step's outcome.  Called by ONE thread per step, as EARLY as the outcome is known (the values are passed
// in, the control-block words themselves are updated when the step closes): the stores travel to page-locked host memory over
// PCIe while the kernel does its work, and are complete when the kernel -- hence the step's completion event -- is.  No fence:
// the host only reads the slot after waiting for that event, and checks the seq word against the step it expects.
DMNIST_DEVICE void publish_status(SyncCtrl* me, uint32_t epoch_after, uint32_t accepted, uint32_t dropped, uint32_t mask,
                                  uint32_t count, uint32_t late) {
  const uint32_t seq = me->status_seq;
  uint32_t* m = me->host_mirror;
  if (m != nullptr) {
    m += 8 * (seq & 3u);
    *reinterpret_cast<uint4*>(m) = make_uint4(epoch_after, me->error, accepted, dropped);
    *reinterpret_cast<uint4*>(m + 4) = make_uint4(mask, count, late, seq + 1);
  }
  me->status_seq = seq + 1;
}

// SGD step size lr(step) / count, as the host schedule (schedule.py) computes it: lr0 * decay_rate^floor(step / decay_steps)
// and the division in double, rounded to fp32 once.  --use_fast_math leaves double precision alone (fp32 would turn the
// power into lg2/ex2.approx and the division into div.approx); CUDA's double pow is within 2 ulp, far below fp32 rounding.
// Thread 0 evaluates it and the CTA reads it after a barrier: every thread of the CTA must call this.
//
// Learning-rate cuts (--lr_plateau_patience): when `cuts` is set and `ctrl` holds a cut table, warp 0 counts the cuts in
// effect at `step` -- c = entries <= step, one relaxed load per lane and a ballot -- and the rate becomes
// lr0 * decay_rate^p * F^c / count, the product in that order in double, as schedule.LearningRateSchedule computes it.
// With c = 0 the factor is 1.0 and the value is the one without a table.  The chief's stores into the table reach every
// replica before any launch whose `step` they concern (DESIGN §4, learning-rate cuts).  Interval mode passes cuts = false.
//
// Learning-rate schedule (--lr_warmup_steps, --lr_cosine_decay_steps): when `ctrl` has one armed, the rate is
// lr0 * D * Wf * F^c / count, left to right, with D = (1 - alpha) * (v * v) + alpha, v = sin(pi * (T - min(s, T)) / (2T))
// in place of decay_rate^p when T > 0, and Wf = f0 + ((1 - f0) * s) / W for s < W.  Every operation of D and Wf is an
// explicitly rounded one: nvcc would contract (1 - alpha) * c + alpha into an FMA the host cannot reproduce.  CUDA's
// double sin is within 2 ulp.  With nothing armed the expression is the one above, unchanged.
DMNIST_DEVICE float cta_scale(const SyncArgs& a, const SyncCtrl* ctrl, bool cuts, uint32_t step, uint32_t count) {
  __shared__ float s_scale;
  if (threadIdx.x < 32) {
    const uint32_t* table = cuts && ctrl != nullptr ? ctrl->lr_cuts : nullptr;
    double f = 1.0;
    if (table != nullptr) {
      const int c = __popc(__ballot_sync(0xffffffffu, ld_relaxed_sys(table + threadIdx.x) <= step));
      if (c > 0) f = pow(ctrl->lr_factor, (double)c);
    }
    if (threadIdx.x == 0) {
      const uint32_t W = ctrl != nullptr ? ctrl->lr_warmup_steps : 0u, T = ctrl != nullptr ? ctrl->lr_cosine_steps : 0u;
      double d;
      if (T > 0) {
        const double q = __ddiv_rn((double)(T - min(step, T)), __dmul_rn(2.0, (double)T));
        const double v = sin(__dmul_rn(3.141592653589793, q));
        const double al = ctrl->lr_cosine_alpha;
        d = __dadd_rn(__dmul_rn(__dadd_rn(1.0, -al), __dmul_rn(v, v)), al);
      } else {
        d = pow(a.decay_rate, (double)(step / (uint32_t)max(a.decay_steps, 1)));
      }
      double lr = a.lr0 * d;
      if (step < W) {
        const double f0 = ctrl->lr_warmup_start;
        lr = __dmul_rn(lr, __dadd_rn(f0, __ddiv_rn(__dmul_rn(__dadd_rn(1.0, -f0), (double)step), (double)W)));
      }
      s_scale = (float)(lr * f / (double)count);
    }
  }
  __syncthreads();
  return s_scale;
}

// Poll (RELAXED loads inside pred) until pred() or the watchdog fires, then ONE acquire load of the flag the wait was about
// (`acq`: LDG.STRONG.SYS + a single CCTL.IVALL; a fence.acq_rel.sys here would be a MEMBAR.ALL.SYS, which also waits for every
// outstanding store of the SM -- and an acquire load on every poll invalidates the SM's
// L1 thousands of times under the co-resident tensor-core kernels).
template <class Pred>
DMNIST_DEVICE bool spin_until(Pred pred, unsigned long long timeout_ns, const volatile uint32_t* acq) {
  bool ok = true;
  if (!pred()) {
    const unsigned long long t0 = globaltimer_ns();
    unsigned spins = 0;
    while (!pred()) {
      if (++spins > 64) {          // busy-poll first (the common wait is a few microseconds), then back off
        __nanosleep(64);
        if ((spins & 255) == 0 && globaltimer_ns() - t0 > timeout_ns) { ok = false; break; }
      }
    }
  }
  (void)ld_acquire_sys(acq);
  return ok;
}

// Device barrier over the ranks of `set` (bit p: rank p; mine may be among them), on the device barrier's words (bar[],
// bar_seq), so that every barrier a replica takes part in, whoever its partners, advances one sequence: local SGD's
// rounds (every rank), gossip SGD's steps (the ring neighbours) and dm_device_barrier.  `P.ctrl` is the table of every
// replica's control block.  Called by one full warp.  Lane p releases my arrival into peer p's block and polls peer p's
// arrival in mine with relaxed loads; spin_until ends every wait with one acquire load of the flag it polled.  Reading a
// peer's data after the barrier needs that acquire: the polls alone order nothing.  Once the warp has synchronised, lane
// 0 adds one system-scope fence, so every lane's acquire is cumulative through it, and the kernel boundary carries it to
// every later kernel of the stream: after this kernel, everything each peer of `set` wrote before its release is
// visible here.  A wait past `timeout_ns` sets the error word to 1.  Returns the nanoseconds spent; `waited` (may be
// null) becomes true when some peer had not yet arrived at the first poll.
template <class Peers>
DMNIST_DEVICE unsigned long long peer_barrier(const Peers& P, SyncCtrl* me, int rank, uint32_t set,
                                              unsigned long long timeout_ns, bool* waited = nullptr) {
  const unsigned long long t0 = globaltimer_ns();
  const uint32_t seq = me->bar_seq + 1;
  bool late = false;
  if (threadIdx.x < SYNC_MAX_RANKS && ((set >> threadIdx.x) & 1u)) {
    st_release_sys(&P.ctrl[threadIdx.x]->bar[rank * 32], seq);
    const volatile uint32_t* flag = &me->bar[threadIdx.x * 32];
    if (waited != nullptr) late = ld_relaxed_sys(flag) < seq;
    if (!spin_until([&] { return ld_relaxed_sys(flag) >= seq; }, timeout_ns, flag)) me->error = 1;
  }
  if (waited != nullptr) *waited = __any_sync(0xffffffffu, late);
  __syncwarp();
  if (threadIdx.x == 0) {
    fence_acq_rel_sys();
    me->bar_seq = seq;
  }
  return globaltimer_ns() - t0;
}

}  // namespace dm
