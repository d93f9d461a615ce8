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

}  // extern "C"
