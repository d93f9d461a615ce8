// Asynchronous SGD (--async_method): TF's asynchronous parameter-server training, on one box.  Every replica free-runs; per
// local iteration
//
//   as_pull_step (1 warp)   r := the chief's update counter (acquire); epoch := r, so the timing rings and the straggler
//                           kernels keep working; stamp t_start
//   as_pull      (grid)     working arena := my master copy (peers add into it: __ldcv), and its bf16 shadow in the same pass
//   <forward / backward of the model on the working arena>
//   as_ticket    (1 warp)   s := atomicAdd_system(&chief->global_step, 1); staleness tau = s - r into the histogram;
//                           publish_status(epoch_after = s + 1)
//   as_apply     (grid)     x = fl(lr(s) * g) (one rounding), then -x added to EVERY replica's master copy: one in-switch
//                           multimem.red on the multicast view, or one red per replica's copy; a system-scope fence ends
//                           every CTA
//
// Nothing is averaged, dropped or waited for: no kernel here reads a word another replica writes in a loop.  The master
// copies are the parameter server's variables, one per replica, each receiving every replica's updates; the working arena
// is private to its replica between iterations, so the live evaluation pass and the live checkpoint capture read one
// pulled state.  Visibility of my own update before my next pull, the end of a run and the bound on extra updates:
// DESIGN.md §4, "Asynchronous SGD".
//
// Stale synchronous parallel (--ssp_staleness=s) adds two 1-warp kernels around that iteration:
//
//   ssp_wait     (1 warp)   before as_pull_step: wait until every peer p that has not retired has clock c_p >= c - s,
//                           c = my clock (updates I have applied); statistics
//   ssp_publish  (1 warp)   after as_apply: c := c + 1, released into line `rank` of every replica's clock board; the
//                           same kernel with 0xFFFFFFFF retires me once my last iteration is enqueued
//
// These are the only async kernels that poll a word another replica writes.  The wait rule, the ordering argument and
// the bounds it gives: DESIGN.md §4, "Stale synchronous parallel".
#include "fused_sync.cuh"

namespace dm {

constexpr int AS_THREADS = 512;
constexpr int AS_BUCKETS = 64;     // staleness histogram: bucket b counts tau = b, the last one tau >= 63
constexpr int AS_LOG = 1024;       // ring of the last (r, s) pairs

// Staleness statistics of one replica, in plain device memory owned by its engine (nobody else writes it).
struct AsyncStats {
  uint32_t hist[AS_BUCKETS];
  unsigned long long tau_sum;
  uint32_t tau_max;
  uint32_t updates;                // updates this replica has applied
  uint32_t pairs[2 * AS_LOG];      // (r, s) of update j at [2 * (j % AS_LOG)]
};
static_assert(sizeof(AsyncStats) == 272 + 8 * AS_LOG, "distributedmnist_b200/parallel/fused.py decodes this layout");

struct AsyncPeers {
  float* master[SYNC_MAX_RANKS];   // every replica's master copy (peer-mapped)
};

DMNIST_DEVICE void red_sys_f32x4(float* p, float4 v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
// In-switch reduction into every replica's copy behind the multicast address.
DMNIST_DEVICE void multimem_red_f32x4(float* mc, float4 v) {
  asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z),
               "f"(v.w)
               : "memory");
}

__global__ void as_pull_step_kernel(SyncCtrl* me, const SyncCtrl* chief) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  const uint32_t r = ld_acquire_sys(&chief->global_step);
  me->as_pull = r;
  me->epoch = r;
  me->t_start[r % TIMING_RING] = globaltimer_ns();
}

__global__ void __launch_bounds__(AS_THREADS) as_pull_kernel(const float* __restrict__ master, float* __restrict__ params,
                                                             __nv_bfloat16* __restrict__ shadow, int numel4) {
  pdl_wait();
  for (int i = blockIdx.x * AS_THREADS + threadIdx.x; i < numel4; i += gridDim.x * AS_THREADS) {
    const float4 v = __ldcv(reinterpret_cast<const float4*>(master) + i);   // peers add into it: not through L1
    reinterpret_cast<float4*>(params)[i] = v;
    if (shadow != nullptr) {
      uint2 o;
      o.x = pack_bf16x2(v.x, v.y);
      o.y = pack_bf16x2(v.z, v.w);
      *reinterpret_cast<uint2*>(shadow + 4 * (size_t)i) = o;
    }
  }
}

__global__ void as_ticket_kernel(SyncCtrl* me, SyncCtrl* chief, AsyncStats* st, int rank) {
  pdl_wait();
  if (threadIdx.x != 0) return;
  const uint32_t s = atomicAdd_system((unsigned int*)&chief->global_step, 1u);
  const uint32_t r = me->as_pull;
  const uint32_t tau = s - r;      // the counter only grows and my ticket is taken after my pull read it: s >= r
  me->as_ticket = s;
  st->hist[min(tau, (uint32_t)(AS_BUCKETS - 1))] += 1;
  st->tau_sum += tau;
  st->tau_max = max(st->tau_max, tau);
  const uint32_t j = st->updates;
  st->pairs[2 * (j % AS_LOG)] = r;
  st->pairs[2 * (j % AS_LOG) + 1] = s;
  st->updates = j + 1;
  me->accepted_steps += 1;
  me->last_mask = 1u << rank;
  me->last_count = 1;
  me->last_late = 0;
  me->t_arrive[r % TIMING_RING] = globaltimer_ns();
  publish_status(me, s + 1, me->accepted_steps, me->dropped_steps, 1u << rank, 1, 0);
}

// -x = -fl(lr(s) * g) into every master copy.  The fence after the CTA's last red makes all of them performed at system
// scope before the kernel completes: the next pull, a later kernel on the same stream, then reads my own update, and the
// end-of-run device barrier, which follows on the stream, releases them to every replica.  With NVLS my own copy is
// reduced through the multicast address while the pull reads it through its unicast one, two virtual aliases of the same
// memory: every thread orders its reductions before later accesses through other aliases with fence.proxy.alias first.
__global__ void __launch_bounds__(AS_THREADS) as_apply_kernel(AsyncPeers P, SyncArgs a, const SyncCtrl* me,
                                                              const float* __restrict__ grads, float* mc_master) {
  pdl_wait();
  const float scale = cta_scale(a, me, false, me->as_ticket, 1u);
  for (int i = blockIdx.x * AS_THREADS + threadIdx.x; i < a.numel4; i += gridDim.x * AS_THREADS) {
    const float4 g = reinterpret_cast<const float4*>(grads)[i];
    float4 x;
    x.x = -__fmul_rn(scale, g.x); x.y = -__fmul_rn(scale, g.y); x.z = -__fmul_rn(scale, g.z); x.w = -__fmul_rn(scale, g.w);
    if (mc_master != nullptr) {
      multimem_red_f32x4(mc_master + 4 * (size_t)i, x);
    } else {
#pragma unroll
      for (int q = 0; q < SYNC_MAX_RANKS; ++q)
        if (q < a.nranks) red_sys_f32x4(P.master[q] + 4 * (size_t)i, x);
    }
  }
  if (mc_master != nullptr) asm volatile("fence.proxy.alias;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) fence_acq_rel_sys();
}

// ---- stale synchronous parallel ---------------------------------------------------------------------------------------
constexpr int SSP_LOG = 1024;                  // ring of the last (c, min peer clock) pairs
constexpr uint32_t SSP_RETIRED = 0xFFFFFFFFu;  // the clock of a replica that has enqueued its last iteration

// Bound statistics and the clock of one replica, in plain device memory owned by its engine (nobody else writes it).
struct SSPStats {
  uint32_t clock;                  // c: updates this replica has applied and published since the bound was armed
  uint32_t waits;                  // iterations whose wait found some peer too far behind
  uint32_t lead_max;               // largest c - (min clock of the non-retired peers) at a pull
  uint32_t pad;
  unsigned long long wait_total_ns;
  unsigned long long wait_max_ns;
  uint32_t pairs[2 * SSP_LOG];     // (c, min non-retired peer clock or 0xFFFFFFFF) of iteration c at [2 * (c % SSP_LOG)]
};
static_assert(sizeof(SSPStats) == 32 + 8 * SSP_LOG, "distributedmnist_b200/parallel/fused.py decodes this layout");

// The clock boards: every replica owns one symmetric board of SYNC_MAX_RANKS 128-byte lines, as SyncCtrl::bar is laid
// out; line p holds peer p's clock.
struct SSPBoards {
  uint32_t* board[SYNC_MAX_RANKS];
};

// Lane p polls peer p's clock in my board with relaxed loads; spin_until ends the wait with one acquire load of it.  The
// predicate c_p + s >= c in 64 bits is c_p >= c - s without a wrap at small c, and always true for a retired peer.  Once
// the warp has synchronised, lane 0's system-scope fence makes every lane's acquire cumulative, and the kernel boundary
// carries it to as_pull_step and as_pull: the pull reads every update each peer applied before it released the clock it
// was seen with (DESIGN.md §4).
__global__ void ssp_wait_kernel(const uint32_t* board, SyncCtrl* me, SSPStats* st, int rank, int nranks, uint32_t s,
                                unsigned long long timeout_ns) {
  pdl_wait();
  const int lane = threadIdx.x;
  const uint32_t c = st->clock;
  const volatile uint32_t* line = board + 32 * lane;
  const bool peer = lane < nranks && lane != rank;
  const auto ready = [&] { return (unsigned long long)ld_relaxed_sys(line) + s >= (unsigned long long)c; };
  const unsigned long long t0 = globaltimer_ns();
  const bool behind = peer && !ready();
  bool ok = true;
  uint32_t seen = SSP_RETIRED;
  if (peer) {
    ok = spin_until(ready, timeout_ns, line);
    seen = ld_relaxed_sys(line);             // >= the value that satisfied the wait: a clock only grows
  }
  const bool waited = __any_sync(0xffffffffu, behind);
  const bool all_ok = __all_sync(0xffffffffu, ok);
  const uint32_t lo = __reduce_min_sync(0xffffffffu, seen);
  if (lane == 0) {
    fence_acq_rel_sys();
    if (!all_ok) me->error = 3;
    if (waited) {
      const unsigned long long ns = globaltimer_ns() - t0;
      st->waits += 1;
      st->wait_total_ns += ns;
      st->wait_max_ns = max(st->wait_max_ns, ns);
    }
    if (lo != SSP_RETIRED && c > lo) st->lead_max = max(st->lead_max, c - lo);
    st->pairs[2 * (c % SSP_LOG)] = c;
    st->pairs[2 * (c % SSP_LOG) + 1] = lo;
  }
}

// c := c + 1 (or the retired value), stored with release semantics into line `rank` of every board.  It follows as_apply
// on the stream, whose CTAs each ended with a system-scope fence (after fence.proxy.alias on the NVLS path): the release
// is ordered after my update has been added to every master copy.
__global__ void ssp_publish_kernel(SSPBoards B, SSPStats* st, int rank, int nranks, int retire) {
  pdl_wait();
  const uint32_t c = retire ? SSP_RETIRED : st->clock + 1u;
  __syncwarp();
  if (threadIdx.x < nranks) st_release_sys(B.board[threadIdx.x] + 32 * rank, c);
  if (threadIdx.x == 0 && !retire) st->clock = c;
}

}  // namespace dm

extern "C" {

int dm_async_stats_bytes() { return (int)sizeof(dm::AsyncStats); }

// First two kernels of an asynchronous iteration: read the update counter from the chief's block (ctrl[0]), then copy my
// master copy into the working arena `params` and its bf16 shadow (null: none).
int dm_async_begin(void* const* ctrl, int rank, const void* master, void* params, void* shadow_bf16, long long numel,
                   int ctas, void* stream_) {
  using namespace dm;
  if (rank < 0 || rank >= SYNC_MAX_RANKS || (numel & 3) || numel / 4 > 0x7fffffffLL) return -1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (ctas < 1 || ctas > num_sms()) ctas = num_sms();
  cudaError_t e = launch_kernel(as_pull_step_kernel, dim3(1), dim3(32), 0, st, reinterpret_cast<SyncCtrl*>(ctrl[rank]),
                                reinterpret_cast<const SyncCtrl*>(ctrl[0]));
  if (e != cudaSuccess) return (int)e;
  return (int)launch_kernel(as_pull_kernel, dim3(ctas), dim3(AS_THREADS), 0, st, reinterpret_cast<const float*>(master),
                            reinterpret_cast<float*>(params), reinterpret_cast<__nv_bfloat16*>(shadow_bf16), (int)(numel / 4));
}

// Last two kernels of an asynchronous iteration: take a ticket from the chief's counter (staleness into `stats`), then add
// -fl(lr(s) * grads) to every replica's master copy -- through the multicast view `mc_master` when it is not null (it must
// then map every copy of the table), else one red per copy of the table `master`.
int dm_async_end(void* const* ctrl, void* const* master, const void* grads, void* stats, int rank, int nranks,
                 long long numel, double lr0, double decay_rate, int decay_steps, int ctas, void* stream_, void* mc_master) {
  using namespace dm;
  if (nranks < 1 || nranks > SYNC_MAX_RANKS || rank < 0 || rank >= nranks || (numel & 3) || numel / 4 > 0x7fffffffLL)
    return -1;
  AsyncPeers P;
  for (int i = 0; i < SYNC_MAX_RANKS; ++i) P.master[i] = reinterpret_cast<float*>(master[i < nranks ? i : rank]);
  SyncArgs a;
  a.rank = rank; a.nranks = nranks; a.k = 1; a.numel4 = (int)(numel / 4);
  a.lr0 = lr0; a.decay_rate = decay_rate; a.decay_steps = decay_steps;
  a.drop_keep = 0.f; a.drop_seed = 0; a.timeout_ns = 0;
  a.shadow = nullptr; a.mc_grads = nullptr; a.mc_params = nullptr;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (ctas < 1 || ctas > num_sms()) ctas = num_sms();
  SyncCtrl* me = reinterpret_cast<SyncCtrl*>(ctrl[rank]);
  cudaError_t e = launch_kernel(as_ticket_kernel, dim3(1), dim3(32), 0, st, me, reinterpret_cast<SyncCtrl*>(ctrl[0]),
                                reinterpret_cast<AsyncStats*>(stats), rank);
  if (e != cudaSuccess) return (int)e;
  return (int)launch_kernel(as_apply_kernel, dim3(ctas), dim3(AS_THREADS), 0, st, P, a, (const SyncCtrl*)me,
                            reinterpret_cast<const float*>(grads), reinterpret_cast<float*>(mc_master));
}

int dm_ssp_stats_bytes() { return (int)sizeof(dm::SSPStats); }

// Stale synchronous parallel, before dm_async_begin: wait until every peer of `nranks` that has not retired has a clock
// of at least c - `s` in my clock board `board` (c: my clock in `stats`).  On a timeout of `timeout_ms` the error word of
// my control block `ctrl` becomes 3.
int dm_ssp_wait(const void* board, void* ctrl, void* stats, int rank, int nranks, unsigned int s, double timeout_ms,
                void* stream_) {
  using namespace dm;
  if (nranks < 1 || nranks > SYNC_MAX_RANKS || rank < 0 || rank >= nranks || s > 0x7fffffffu || board == nullptr ||
      ctrl == nullptr || stats == nullptr)
    return -1;
  return (int)launch_kernel(ssp_wait_kernel, dim3(1), dim3(32), 0, reinterpret_cast<cudaStream_t>(stream_),
                            reinterpret_cast<const uint32_t*>(board), reinterpret_cast<SyncCtrl*>(ctrl),
                            reinterpret_cast<SSPStats*>(stats), rank, nranks, s,
                            (unsigned long long)(timeout_ms * 1e6));
}

// After dm_async_end: advance my clock in `stats` and publish it into every board of the table `boards`; `retire` != 0
// publishes the retired value 0xFFFFFFFF instead and leaves the clock alone.
int dm_ssp_publish(void* const* boards, void* stats, int rank, int nranks, int retire, void* stream_) {
  using namespace dm;
  if (nranks < 1 || nranks > SYNC_MAX_RANKS || rank < 0 || rank >= nranks || stats == nullptr) return -1;
  SSPBoards B;
  for (int i = 0; i < SYNC_MAX_RANKS; ++i) B.board[i] = reinterpret_cast<uint32_t*>(boards[i < nranks ? i : rank]);
  return (int)launch_kernel(ssp_publish_kernel, dim3(1), dim3(32), 0, reinterpret_cast<cudaStream_t>(stream_), B,
                            reinterpret_cast<SSPStats*>(stats), rank, nranks, retire);
}

}  // extern "C"
