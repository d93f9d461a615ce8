// Local SGD (--local_sgd_steps=H), also called periodic model averaging: every replica applies its own gradient to its
// own weights, and every H global steps the replicas replace their weights with the mean of all copies.  Per iteration
//
//   ls_apply  (grid)     w := w - fp32(lr(s)) * g (one FFMA), bf16 shadow := RNE(w); s = the epoch word; stamps t_arrive
//   ls_enter  (1 warp)   epoch := s + 1; if (s + 1) % H == 0: barrier "every replica's step s is applied"
//   ls_average (grid)    if averaging: owner q of shard q writes fl(S / N) into shard q of EVERY replica's arena
//   ls_leave  (1 warp)   if averaging: barrier "every shard of every arena holds the average"; statistics; status
//   ls_shadow (grid)     if averaging: bf16 shadow := RNE(my arena)
//
// A step that is not an averaging step runs ls_apply and four kernels that return at once: the predicate is evaluated
// on the device from the epoch word, so one captured graph per input slot serves every step (DESIGN.md §4, "Local
// SGD").  Only the two barriers wait on another replica; ls_average's arithmetic reads and writes shard q alone, so a
// single process can run it for every q over N arenas on one GPU.
#include "fused_sync.cuh"

namespace dm {

constexpr int LS_THREADS = 512;

// Averaging statistics of one replica, in plain device memory owned by its engine (nobody else writes it).
struct LocalStats {
  uint32_t rounds;                   // averaging rounds completed
  uint32_t pad;
  unsigned long long wait_total_ns;  // %globaltimer ns spent in both barriers of every round
  unsigned long long wait_max_ns;    // the longest round's two barriers
  unsigned long long wait_enter_ns;  // the current round's first barrier (until ls_leave adds it up)
};
static_assert(sizeof(LocalStats) == 32, "distributedmnist_b200/parallel/fused.py decodes this layout");

struct LocalPeers {
  SyncCtrl* ctrl[SYNC_MAX_RANKS];
  float* params[SYNC_MAX_RANKS];     // every replica's arena (peer-mapped)
};

DMNIST_DEVICE bool averaging_step(const SyncCtrl* me, uint32_t period) { return me->epoch % period == 0u; }

// The barrier of both rounds' sides: peer_barrier (fused_sync.cuh) over every rank, on the device barrier's words, so
// that it and dm_device_barrier keep one sequence: every replica runs the same steps, hence the same barriers in the same
// order.  Returns the nanoseconds spent.
DMNIST_DEVICE unsigned long long ls_barrier(const LocalPeers& P, SyncCtrl* me, int rank, int nranks,
                                            unsigned long long timeout_ns) {
  return peer_barrier(P, me, rank, (1u << nranks) - 1u, timeout_ns);
}

__global__ void __launch_bounds__(LS_THREADS) ls_apply_kernel(SyncArgs a, SyncCtrl* me, const float* __restrict__ grads,
                                                              float* __restrict__ params, uint32_t period) {
  pdl_wait();
  const uint32_t s = me->epoch;
  if (blockIdx.x == 0 && threadIdx.x == 0) me->t_arrive[s % TIMING_RING] = globaltimer_ns();   // gradient complete
  const float scale = cta_scale(a, me, false, s, 1u);
  for (int i = blockIdx.x * LS_THREADS + threadIdx.x; i < a.numel4; i += gridDim.x * LS_THREADS) {
    const float4 g = reinterpret_cast<const float4*>(grads)[i];
    float4 w = reinterpret_cast<const float4*>(params)[i];
    w.x -= scale * g.x; w.y -= scale * g.y; w.z -= scale * g.z; w.w -= scale * g.w;     // one FFMA each
    reinterpret_cast<float4*>(params)[i] = w;
    if (a.shadow != nullptr) {
      uint2 o;
      o.x = pack_bf16x2(w.x, w.y);
      o.y = pack_bf16x2(w.z, w.w);
      *reinterpret_cast<uint2*>(a.shadow + 4 * (size_t)i) = o;
    }
  }
  // Before an averaging round: the fence makes this CTA's new weights performed at system scope before the kernel
  // completes, so ls_enter's release, which follows on the stream, publishes them to every peer's ls_average.  With NVLS
  // those peers read my arena through the multicast address: fence.proxy.alias orders my unicast stores first.
  if ((s + 1u) % period == 0u) {
    if (a.mc_params != nullptr) asm volatile("fence.proxy.alias;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0) fence_acq_rel_sys();
  }
}

__global__ void ls_enter_kernel(LocalPeers P, LocalStats* st, int rank, int nranks, uint32_t period, int close,
                                unsigned long long timeout_ns) {
  pdl_wait();
  SyncCtrl* me = P.ctrl[rank];
  if (threadIdx.x == 0 && close) {
    me->epoch = me->epoch + 1u;            // the global step of my weights: every replica makes one step per global step
    me->accepted_steps += 1;
    me->last_mask = 1u << rank;
    me->last_count = 1;
    me->last_late = 0;
  }
  __syncwarp();
  if (!averaging_step(me, period)) return;
  const unsigned long long ns = ls_barrier(P, me, rank, nranks, timeout_ns);
  if (threadIdx.x == 0) st->wait_enter_ns = ns;
}

// Owner `rank` of shard [rank * chunk, (rank + 1) * chunk) (float4 units): w = fl(S / N) into that shard of every arena.
// Peer path: S summed from +0.0 in rank order, one load per copy, and stored into every copy.  NVLS (`mc` not null, the
// multicast view of the arenas): one multimem.ld_reduce returns S summed in the switch's order, one multimem.st lands w
// in every copy.  The arithmetic reads and writes the owner's shard only and waits on nobody.
__global__ void __launch_bounds__(LS_THREADS) ls_average_kernel(LocalPeers P, const SyncCtrl* me, int rank, int nranks,
                                                                int numel4, uint32_t period, float* mc) {
  pdl_wait();
  if (!averaging_step(me, period)) return;
  const int chunk = (numel4 + nranks - 1) / nranks;
  const int lo = rank * chunk, hi = min(numel4, lo + chunk);
  const float n = (float)nranks;
  for (int i = lo + blockIdx.x * LS_THREADS + threadIdx.x; i < hi; i += gridDim.x * LS_THREADS) {
    float4 s;
    if (mc != nullptr) {
      s = multimem_ld_reduce_f4(mc + 4 * (size_t)i);
    } else {
      s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int q = 0; q < SYNC_MAX_RANKS; ++q)
        if (q < nranks) {
          const float4 v = ld_peer_f4(P.params[q] + 4 * (size_t)i);
          s.x = __fadd_rn(s.x, v.x); s.y = __fadd_rn(s.y, v.y); s.z = __fadd_rn(s.z, v.z); s.w = __fadd_rn(s.w, v.w);
        }
    }
    const float4 w = make_float4(__fdiv_rn(s.x, n), __fdiv_rn(s.y, n), __fdiv_rn(s.z, n), __fdiv_rn(s.w, n));
    if (mc != nullptr) {
      multimem_st_f4(mc + 4 * (size_t)i, w);
    } else {
#pragma unroll
      for (int q = 0; q < SYNC_MAX_RANKS; ++q)
        if (q < nranks) st_peer_f4(P.params[q] + 4 * (size_t)i, w);
    }
  }
  // The average was written through the multicast address (NVLS) and is read later through unicast ones (ls_shadow, the
  // next step): fence.proxy.alias orders the two aliases.  The system-scope fence makes every store performed before the
  // kernel completes, so ls_leave's release publishes them.
  if (mc != nullptr) asm volatile("fence.proxy.alias;" ::: "memory");
  __syncthreads();
  if (threadIdx.x == 0) fence_acq_rel_sys();
}

__global__ void ls_leave_kernel(LocalPeers P, LocalStats* st, int rank, int nranks, uint32_t period, int close,
                                unsigned long long timeout_ns) {
  pdl_wait();
  SyncCtrl* me = P.ctrl[rank];
  if (averaging_step(me, period)) {
    const unsigned long long ns = ls_barrier(P, me, rank, nranks, timeout_ns);
    if (threadIdx.x == 0) {
      const unsigned long long round = st->wait_enter_ns + ns;
      st->rounds += 1;
      st->wait_total_ns += round;
      st->wait_max_ns = max(st->wait_max_ns, round);
    }
  }
  if (threadIdx.x == 0 && close)
    publish_status(me, me->epoch, me->accepted_steps, me->dropped_steps, 1u << rank, 1, 0);
}

__global__ void __launch_bounds__(LS_THREADS) ls_shadow_kernel(const SyncCtrl* me, const float* params,
                                                               __nv_bfloat16* __restrict__ shadow, int numel4,
                                                               uint32_t period) {
  pdl_wait();
  if (!averaging_step(me, period)) return;
  for (int i = blockIdx.x * LS_THREADS + threadIdx.x; i < numel4; i += gridDim.x * LS_THREADS) {
    const float4 v = __ldcv(reinterpret_cast<const float4*>(params) + i);    // peers stored into it: not through L1
    uint2 o;
    o.x = pack_bf16x2(v.x, v.y);
    o.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(shadow + 4 * (size_t)i) = o;
  }
}

}  // namespace dm

extern "C" {

int dm_local_stats_bytes() { return (int)sizeof(dm::LocalStats); }

// The local update of one iteration: params -= fp32(lr(s)) * grads and the bf16 shadow (null: none), s = the epoch
// word of my block (ctrl[rank]), with the block's learning-rate schedule.  `period` = H names the averaging steps, before
// which the kernel ends with a system-scope fence (and, when `mc_params` is not null, a proxy fence).
int dm_local_apply(void* const* ctrl, int rank, void* params, const void* grads, void* shadow_bf16, long long numel,
                   unsigned int period, double lr0, double decay_rate, int decay_steps, int ctas, void* stream_,
                   const void* mc_params) {
  using namespace dm;
  if (rank < 0 || rank >= SYNC_MAX_RANKS || period < 1 || (numel & 3) || numel / 4 > 0x7fffffffLL) return -1;
  SyncArgs a;
  a.rank = rank; a.nranks = 1; a.k = 1; a.numel4 = (int)(numel / 4);
  a.lr0 = lr0; a.decay_rate = decay_rate; a.decay_steps = decay_steps;
  a.drop_keep = 0.f; a.drop_seed = 0; a.timeout_ns = 0;
  a.shadow = reinterpret_cast<__nv_bfloat16*>(shadow_bf16);
  a.mc_grads = nullptr;
  a.mc_params = const_cast<float*>(reinterpret_cast<const float*>(mc_params));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (ctas < 1 || ctas > num_sms()) ctas = num_sms();
  return (int)launch_kernel(ls_apply_kernel, dim3(ctas), dim3(LS_THREADS), 0, st, a, reinterpret_cast<SyncCtrl*>(ctrl[rank]),
                            reinterpret_cast<const float*>(grads), reinterpret_cast<float*>(params), period);
}

// The averaging round of one iteration, after dm_local_apply: enter (with `close`: the step is closed, epoch + 1),
// average, leave (with `close`: the step's status is published), shadow.  Each kernel acts only when the epoch word is a
// multiple of `period`; `close` = 0 with `period` = 1 is the unconditional round that ends a run.  `params` is the table
// of every replica's arena, `mc_params` its multicast view or null (peer path), `stats` dm_local_stats_bytes() bytes.
int dm_local_average(void* const* ctrl, void* const* params, void* shadow_bf16, void* stats, int rank, int nranks,
                     long long numel, unsigned int period, int close, double timeout_ms, int ctas, void* stream_,
                     void* mc_params) {
  using namespace dm;
  if (nranks < 1 || nranks > SYNC_MAX_RANKS || rank < 0 || rank >= nranks || period < 1 || (numel & 3) ||
      numel / 4 > 0x7fffffffLL || shadow_bf16 == nullptr || stats == nullptr)
    return -1;
  LocalPeers P;
  for (int i = 0; i < SYNC_MAX_RANKS; ++i) {
    const int j = i < nranks ? i : rank;
    P.ctrl[i] = reinterpret_cast<SyncCtrl*>(ctrl[j]);
    P.params[i] = reinterpret_cast<float*>(params[j]);
  }
  LocalStats* s = reinterpret_cast<LocalStats*>(stats);
  const unsigned long long tns = (unsigned long long)(timeout_ms * 1e6);
  const int numel4 = (int)(numel / 4);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (ctas < 1 || ctas > num_sms()) ctas = num_sms();
  SyncCtrl* me = P.ctrl[rank];
  cudaError_t e = launch_kernel(ls_enter_kernel, dim3(1), dim3(32), 0, st, P, s, rank, nranks, period, close, tns);
  if (e != cudaSuccess) return (int)e;
  e = launch_kernel(ls_average_kernel, dim3(ctas), dim3(LS_THREADS), 0, st, P, (const SyncCtrl*)me, rank, nranks, numel4,
                    period, reinterpret_cast<float*>(mc_params));
  if (e != cudaSuccess) return (int)e;
  e = launch_kernel(ls_leave_kernel, dim3(1), dim3(32), 0, st, P, s, rank, nranks, period, close, tns);
  if (e != cudaSuccess) return (int)e;
  return (int)launch_kernel(ls_shadow_kernel, dim3(ctas), dim3(LS_THREADS), 0, st, (const SyncCtrl*)me,
                            (const float*)P.params[rank], reinterpret_cast<__nv_bfloat16*>(shadow_bf16), numel4, period);
}

// ls_average_kernel alone, for shard owner `rank` of `nranks` arenas (`params`, a table of device pointers that may all
// live on this GPU), with no barrier around it: the averaging arithmetic, for checks.  Acts when ctrl's epoch word is a
// multiple of `period`.
int dm_local_average_shard(const void* ctrl, void* const* params, int rank, int nranks, long long numel,
                           unsigned int period, int ctas, void* stream_, void* mc_params) {
  using namespace dm;
  if (nranks < 1 || nranks > SYNC_MAX_RANKS || rank < 0 || rank >= nranks || period < 1 || (numel & 3) ||
      numel / 4 > 0x7fffffffLL)
    return -1;
  LocalPeers P;
  for (int i = 0; i < SYNC_MAX_RANKS; ++i) {
    P.ctrl[i] = nullptr;
    P.params[i] = reinterpret_cast<float*>(params[i < nranks ? i : rank]);
  }
  if (ctas < 1 || ctas > num_sms()) ctas = num_sms();
  return (int)launch_kernel(ls_average_kernel, dim3(ctas), dim3(LS_THREADS), 0, reinterpret_cast<cudaStream_t>(stream_), P,
                            reinterpret_cast<const SyncCtrl*>(ctrl), rank, nranks, (int)(numel / 4), period,
                            reinterpret_cast<float*>(mc_params));
}

}  // extern "C"
