// Consistent snapshot of the chief's parameter arena for the in-training validation pass when peers may push weights into
// that arena at any time (K < N backup workers, interval mode).  engine_cuda.CudaLeNetEngine.arm_eval(snapshot=True)
// captures R attempts in front of the pass; each attempt is three launches, whose boundaries are the grid barriers:
//
//   snap_select    1 warp   newest committed step g: start at global_step, walk forward while commit[g % RING] carries tag
//                           g + 1; wait (short watchdog) until g's writers released done >= g, moving on to a newer commit
//                           if one appears meanwhile.  Tag of commit[(g - 1) % RING] below g: nothing of g is in flight
//                           (checkpoint restore, nothing committed yet).
//   snap_copy      grid     fp32 arena -> snapshot (loads bypass L1), bf16 shadow of the ranges the pass reads with
//                           f32_to_bf16_kernel's packing; every CTA fences (fence.acq_rel.sys) after its loads.
//   snap_validate  1 warp   commit[g % RING] -- the slot of step g + 1 -- holds a tag > g: a push of a newer step may have
//                           overlapped the copy, the attempt fails.  Otherwise the snapshot holds exactly step g.
//   snap_keep      grid     optional, after the attempts: copy an accepted snapshot aside (a later pass's failed attempt
//                           overwrites the snapshot buffer), so the last accepted one stays readable.
//
// Why that suffices (DESIGN §4.4): every push of step g happens after the CAS that puts tag g into commit[(g - 1) % RING];
// `done` of g's writers is released after a system fence covering all their pushes; steps commit in order and tags are full
// step numbers.  So after the done wait every element holds step g or newer, and a copy that read any element of step g + 1
// or later ran after the CAS of tag g + 1, which validate then sees.  Only words the aggregation kernels already write are
// read.  The pushes themselves are weak st.global stores: like every aggregation kernel, the argument relies on the
// message-passing order csrc/litmus.cu exercises.
//
// Also here, for the tests only: a peer emulation (commit word -> pushes of f(g, i) -> done, in either mode's order) and a
// paced single-CTA writer that runs next to the snapshot on another stream.
#include "fused_sync.cuh"

namespace dm {

constexpr int SNAP_THREADS = 512;

struct SnapState {
  uint32_t step;              // step of the newest accepted snapshot (the pass's record reports it)
  int32_t status;             // this pass: 0 = nothing accepted yet, n > 0 = attempt n accepted, -1 = no consistent snapshot
  uint32_t cand;              // this attempt's candidate step
  uint32_t cand_ok;           // 1: select found the candidate's pushes complete
  uint32_t attempts;          // statistics since the state was zeroed
  uint32_t rejected;          // validate saw a newer commit
  uint32_t timeouts;          // select's watchdog fired
  uint32_t accepted_passes;
  uint32_t failed_passes;
  uint32_t laps;              // select found the slot of its step already reused (a ring lap behind)
  uint32_t keep_step;         // step of the kept copy (snap_keep), 0xffffffff: none kept yet
  uint32_t pad[5];
};

DMNIST_DEVICE unsigned long long commit_word(const SyncCtrl* c, uint32_t slot_step) {
  return ld_acquire_sys64(reinterpret_cast<const volatile unsigned long long*>(&c->commit[slot_step % SYNC_RING]));
}

// newest committed step reachable from g by following the tags
DMNIST_DEVICE uint32_t walk_commits(const SyncCtrl* c, uint32_t g) {
  for (int n = 0; n < SYNC_RING; ++n) {
    if ((uint32_t)(commit_word(c, g) >> 32) != g + 1) break;
    ++g;
  }
  return g;
}

DMNIST_DEVICE void snap_fail(SnapState* s) {
  s->status = -1;
  s->failed_passes += 1;
}

__global__ void snap_select_kernel(const SyncCtrl* c, SnapState* s, int attempt, int interval,
                                   unsigned long long watchdog_ns) {
  if (threadIdx.x != 0) return;
  if (attempt == 0) s->status = 0;
  if (s->status != 0) return;                       // an earlier attempt of this pass was accepted
  s->attempts += 1;
  s->cand_ok = 0;
  uint32_t g = walk_commits(c, ld_acquire_sys(&c->global_step));
  const unsigned long long t0 = globaltimer_ns();
  for (;;) {
    if (g == 0) break;                              // nothing committed: the initial weights
    const unsigned long long cw = commit_word(c, g - 1);
    const uint32_t tag = (uint32_t)(cw >> 32);
    if (tag < g) break;                             // restored step: its weights were written by the host, nothing pending
    if (tag > g) { s->cand = g; s->laps += 1; return; }       // slot already reused: a ring lap behind, attempt fails
    const uint32_t writers = interval ? (1u << (((uint32_t)cw >> 8) & 0xffu)) : ((uint32_t)cw & 0xffu);
    bool landed = true;
    for (int q = 0; q < SYNC_MAX_RANKS; ++q)
      if (((writers >> q) & 1u) && ld_relaxed_sys(&c->done[q * 32]) < g) landed = false;
    if (landed) {
      fence_acq_rel_sys();                          // acquire side of the writers' done releases
      break;
    }
    if (globaltimer_ns() - t0 > watchdog_ns) { s->cand = g; s->timeouts += 1; return; }
    __nanosleep(256);
    g = walk_commits(c, g);                         // a newer commit appeared: score that one instead
  }
  s->cand = g;
  s->cand_ok = 1;
}

__global__ void __launch_bounds__(SNAP_THREADS) snap_copy_kernel(const SnapState* s, const float* __restrict__ params,
                                                                 float* __restrict__ snap, __nv_bfloat16* __restrict__ snap16,
                                                                 int numel4, int4 bf_ranges) {
  if (s->status != 0 || !s->cand_ok) return;
  for (int i = blockIdx.x * SNAP_THREADS + threadIdx.x; i < numel4; i += gridDim.x * SNAP_THREADS) {
    const float4 v = __ldcv(reinterpret_cast<const float4*>(params) + i);   // peers push into this arena: not through L1
    reinterpret_cast<float4*>(snap)[i] = v;
    if ((i >= bf_ranges.x && i < bf_ranges.y) || (i >= bf_ranges.z && i < bf_ranges.w)) {
      uint2 o;
      o.x = pack_bf16x2(v.x, v.y);
      o.y = pack_bf16x2(v.z, v.w);
      reinterpret_cast<uint2*>(snap16)[i] = o;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) fence_acq_rel_sys();        // this CTA's loads are ordered before validate's commit-word read
}

__global__ void snap_validate_kernel(const SyncCtrl* c, SnapState* s, int attempt, int attempts) {
  if (threadIdx.x != 0) return;
  if (s->status != 0) return;
  const bool last = attempt == attempts - 1;
  if (!s->cand_ok) {
    if (last) snap_fail(s);
    return;
  }
  const uint32_t g = s->cand;
  if ((uint32_t)(commit_word(c, g) >> 32) > g) {    // step g + 1 (or a later lap) committed: pushes may have overlapped
    s->rejected += 1;
    if (last) snap_fail(s);
    return;
  }
  s->step = g;
  s->status = attempt + 1;
  s->accepted_passes += 1;
}

// Optional, after the attempts of a pass: keep a copy of an accepted snapshot, which a later failed attempt would overwrite.
__global__ void __launch_bounds__(SNAP_THREADS) snap_keep_kernel(SnapState* s, const float* __restrict__ snap,
                                                                 float* __restrict__ keep, int numel4) {
  if (s->status <= 0) return;
  for (int i = blockIdx.x * SNAP_THREADS + threadIdx.x; i < numel4; i += gridDim.x * SNAP_THREADS)
    reinterpret_cast<float4*>(keep)[i] = reinterpret_cast<const float4*>(snap)[i];
  if (blockIdx.x == 0 && threadIdx.x == 0) s->keep_step = s->step;
}

// ---- test support: a peer that commits step g and pushes f(g, i) into the chief's arena ----------------------------------
DMNIST_DEVICE float snap_test_value(uint32_t g, int i) { return (float)g + (float)(i & 1023) * (1.0f / 1024.0f); }

// The whole CTA.  phases: 1 = commit word, 2 = pushes, 4 = done.  K < N order: commit, global_step, pushes, done; interval
// order: commit, pushes, global_step, done.  The emulated writer is rank `writer` (mask bit, committer field, done slot).
DMNIST_DEVICE void emulate_round(SyncCtrl* c, float* params, int numel, uint32_t g, int interval, int writer, int phases) {
  const unsigned long long cw = ((unsigned long long)g << 32) |
                                (interval ? ((unsigned long long)writer << 8) : 0ull) | (1ull << writer);
  if ((phases & 1) && threadIdx.x == 0) {
    atomicExch(reinterpret_cast<unsigned long long*>(&c->commit[(g - 1) % SYNC_RING]), cw);
    __threadfence_system();
    if (!interval) atomicMax((unsigned int*)&c->global_step, g);
    __threadfence_system();
  }
  __syncthreads();
  if (phases & 2)
    for (int i = threadIdx.x; i < numel; i += blockDim.x) params[i] = snap_test_value(g, i);
  __syncthreads();
  if ((phases & 4) && threadIdx.x == 0) {
    __threadfence_system();
    if (interval) atomicMax((unsigned int*)&c->global_step, g);
    __threadfence_system();
    st_release_sys(&c->done[writer * 32], g);
  }
  __syncthreads();
}

__global__ void snap_emulate_kernel(SyncCtrl* c, float* params, int numel, uint32_t g, int interval, int writer, int phases) {
  emulate_round(c, params, numel, g, interval, writer, phases);
}

// Paced writer for the concurrent test: raises *host_flag = 1 once resident, then commits rounds g0 + 1 .. g0 + rounds, each
// followed by a pause of pace_ns, and raises *host_flag = 2 at the end.  It never waits for the reader.
__global__ void snap_writer_kernel(SyncCtrl* c, float* params, int numel, uint32_t g0, int rounds, unsigned long long pace_ns,
                                   int interval, volatile uint32_t* host_flag) {
  if (threadIdx.x == 0) { *host_flag = 1u; __threadfence_system(); }
  for (int r = 1; r <= rounds; ++r) {
    emulate_round(c, params, numel, g0 + (uint32_t)r, interval, 1, 7);
    if (threadIdx.x == 0) {
      const unsigned long long t0 = globaltimer_ns();
      while (globaltimer_ns() - t0 < pace_ns) __nanosleep(500);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { __threadfence_system(); *host_flag = 2u; }
}

}  // namespace dm

extern "C" {

int dm_snap_state_bytes() { return (int)sizeof(dm::SnapState); }

// One snapshot attempt (select, copy, validate) of a pass of `attempts`.  ctrl: the chief's control block; bf ranges: two
// [begin, end) float ranges (multiples of 4) whose bf16 shadow the pass reads.
int dm_snap_select(const void* ctrl, void* state, int attempt, int interval, double watchdog_ms, void* stream) {
  dm::snap_select_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const dm::SyncCtrl*>(ctrl), reinterpret_cast<dm::SnapState*>(state), attempt, interval,
      (unsigned long long)(watchdog_ms * 1e6));
  return (int)cudaGetLastError();
}

int dm_snap_copy(const void* state, const void* params, void* snap, void* snap_bf16, long long numel, long long r0b,
                 long long r0e, long long r1b, long long r1e, void* stream) {
  if ((numel | r0b | r0e | r1b | r1e) & 3) return -1;
  const int4 rg = make_int4((int)(r0b / 4), (int)(r0e / 4), (int)(r1b / 4), (int)(r1e / 4));
  dm::snap_copy_kernel<<<dm::num_sms(), dm::SNAP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const dm::SnapState*>(state), reinterpret_cast<const float*>(params), reinterpret_cast<float*>(snap),
      reinterpret_cast<__nv_bfloat16*>(snap_bf16), (int)(numel / 4), rg);
  return (int)cudaGetLastError();
}

int dm_snap_validate(const void* ctrl, void* state, int attempt, int attempts, void* stream) {
  dm::snap_validate_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const dm::SyncCtrl*>(ctrl), reinterpret_cast<dm::SnapState*>(state), attempt, attempts);
  return (int)cudaGetLastError();
}

int dm_snap_keep(void* state, const void* snap, void* keep, long long numel, void* stream) {
  if (numel & 3) return -1;
  dm::snap_keep_kernel<<<dm::num_sms(), dm::SNAP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<dm::SnapState*>(state), reinterpret_cast<const float*>(snap), reinterpret_cast<float*>(keep),
      (int)(numel / 4));
  return (int)cudaGetLastError();
}

// Test support (see above).
int dm_snap_test_emulate(void* ctrl, void* params, long long numel, unsigned int g, int interval, int writer, int phases,
                         void* stream) {
  if (g == 0 || writer < 0 || writer >= dm::SYNC_MAX_RANKS) return -1;
  dm::snap_emulate_kernel<<<1, 1024, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<dm::SyncCtrl*>(ctrl), reinterpret_cast<float*>(params), (int)numel, g, interval, writer, phases);
  return (int)cudaGetLastError();
}

int dm_snap_test_writer(void* ctrl, void* params, long long numel, unsigned int g0, int rounds, double pace_us, int interval,
                        void* host_flag, void* stream) {
  dm::snap_writer_kernel<<<1, 1024, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<dm::SyncCtrl*>(ctrl), reinterpret_cast<float*>(params), (int)numel, g0, rounds,
      (unsigned long long)(pace_us * 1e3), interval, reinterpret_cast<volatile uint32_t*>(host_flag));
  return (int)cudaGetLastError();
}

}  // extern "C"
