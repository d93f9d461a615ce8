// Gossip SGD (--gossip_method), decentralized SGD on a ring: every step each replica averages its half step with those of
// its two ring neighbours, and waits for those two only.  Adapt-then-combine, w := W (w - lr g) with the doubly
// stochastic ring matrix W of weight 1/m, m = |N(i)| = min(N, 3), N(i) = {i - 1, i, i + 1} mod N.  Per iteration
//
//   gs_apply   (grid)    h = w - fp32(lr(s)) * g (one FFMA) into my send buffer send_i[s % 2]; s = the epoch word; stamps
//                        t_arrive; ends with a system-scope fence.  The arena is not written.
//   gs_barrier (1 warp)  closes the step (epoch := s + 1, accepted, status); peer_barrier over N(i): releases my arrival
//                        to my two neighbours, polls theirs; statistics and the %globaltimer time it passed
//   gs_mix     (grid)    w = fl(S / m), S = the sum of send_j[s % 2] over N(i) from +0.0 in increasing rank order
//                        (peer loads, __fadd_rn), the division __fdiv_rn; bf16 shadow := RNE(w)
//
// One barrier per iteration is enough because the send buffers alternate: replica j overwrites send_j[s % 2] only in its
// apply of iteration s + 2, after it passed its barrier of s + 1, which needs my release of s + 1, which my stream issues
// after my gs_mix(s) has completed (DESIGN.md §4, "Gossip SGD").  No peer reads or writes a replica's arena.  For N <= 3,
// N(i) is every rank and gs_mix sums the terms ls_average_kernel sums, in the same order: gossip SGD is then bit for bit
// --local_sgd_steps=1 on the peer path.
#include "fused_sync.cuh"

namespace dm {

constexpr int GS_THREADS = 512;

// Statistics of one replica, in plain device memory owned by its engine (nobody else writes it).
struct GossipStats {
  uint32_t iterations;               // barriers passed (one per iteration)
  uint32_t waits;                    // barriers at whose first poll some neighbour had not yet arrived
  unsigned long long wait_total_ns;  // %globaltimer ns spent in the barriers
  unsigned long long wait_max_ns;    // the longest one
  unsigned long long pad;
  unsigned long long t_pass[TIMING_RING];   // %globaltimer when the barrier of iteration s was passed, at [s % RING]
};
static_assert(sizeof(GossipStats) == 32 + 8 * TIMING_RING, "distributedmnist_b200/parallel/fused.py decodes this layout");

struct GossipPeers {
  SyncCtrl* ctrl[SYNC_MAX_RANKS];
  const float* send[SYNC_MAX_RANKS];   // every replica's send buffers, 2 x numel fp32 each (peer-mapped)
};

// N(rank) as a rank mask: {rank - 1, rank, rank + 1} mod nranks.  Every rank for nranks <= 3.
DMNIST_DEVICE uint32_t ring_set(int rank, int nranks) {
  return (1u << rank) | (1u << ((rank + 1) % nranks)) | (1u << ((rank + nranks - 1) % nranks));
}

__global__ void __launch_bounds__(GS_THREADS) gs_apply_kernel(SyncArgs a, SyncCtrl* me, const float* __restrict__ grads,
                                                              const float* __restrict__ params, float* __restrict__ send) {
  pdl_wait();
  const uint32_t s = me->epoch;
  if (blockIdx.x == 0 && threadIdx.x == 0) me->t_arrive[s % TIMING_RING] = globaltimer_ns();   // gradient complete
  const float scale = cta_scale(a, me, false, s, 1u);
  float4* h = reinterpret_cast<float4*>(send) + (size_t)(s & 1u) * a.numel4;
  for (int i = blockIdx.x * GS_THREADS + threadIdx.x; i < a.numel4; i += gridDim.x * GS_THREADS) {
    const float4 g = reinterpret_cast<const float4*>(grads)[i];
    float4 w = reinterpret_cast<const float4*>(params)[i];
    w.x -= scale * g.x; w.y -= scale * g.y; w.z -= scale * g.z; w.w -= scale * g.w;     // one FFMA each, as ls_apply
    h[i] = w;
  }
  // the half step is performed at system scope before the kernel completes, so gs_barrier's release, which follows on
  // the stream, publishes it to both neighbours' gs_mix
  __syncthreads();
  if (threadIdx.x == 0) fence_acq_rel_sys();
}

__global__ void gs_barrier_kernel(GossipPeers P, GossipStats* st, int rank, int nranks, unsigned long long timeout_ns) {
  pdl_wait();
  SyncCtrl* me = P.ctrl[rank];
  const uint32_t s = me->epoch;
  if (threadIdx.x == 0) {
    me->epoch = s + 1u;                    // my iteration count, which is the global step of my weights
    me->accepted_steps += 1;
    me->last_mask = 1u << rank;
    me->last_count = 1;
    me->last_late = 0;
  }
  __syncwarp();
  bool waited;
  const unsigned long long ns = peer_barrier(P, me, rank, ring_set(rank, nranks), timeout_ns, &waited);
  if (threadIdx.x == 0) {
    st->t_pass[s % TIMING_RING] = globaltimer_ns();
    st->iterations += 1;
    st->waits += waited ? 1u : 0u;
    st->wait_total_ns += ns;
    st->wait_max_ns = max(st->wait_max_ns, ns);
    publish_status(me, s + 1u, me->accepted_steps, me->dropped_steps, 1u << rank, 1, 0);
  }
}

// After gs_barrier: the epoch word is s + 1.  Every load of a neighbour's send buffer feeds a store of this kernel, so all
// of them have returned when it completes, before gs_barrier of s + 1 releases the neighbour to overwrite the buffer.
__global__ void __launch_bounds__(GS_THREADS) gs_mix_kernel(GossipPeers P, const SyncCtrl* me, int rank, int nranks,
                                                            int numel4, float* __restrict__ params,
                                                            __nv_bfloat16* __restrict__ shadow) {
  pdl_wait();
  const size_t off = (size_t)((me->epoch - 1u) & 1u) * numel4;
  const uint32_t set = ring_set(rank, nranks);
  const float m = (float)__popc(set);
  for (int i = blockIdx.x * GS_THREADS + threadIdx.x; i < numel4; i += gridDim.x * GS_THREADS) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int q = 0; q < SYNC_MAX_RANKS; ++q)
      if ((set >> q) & 1u) {
        const float4 v = ld_peer_f4(P.send[q] + 4 * (off + i));
        s.x = __fadd_rn(s.x, v.x); s.y = __fadd_rn(s.y, v.y); s.z = __fadd_rn(s.z, v.z); s.w = __fadd_rn(s.w, v.w);
      }
    const float4 w = make_float4(__fdiv_rn(s.x, m), __fdiv_rn(s.y, m), __fdiv_rn(s.z, m), __fdiv_rn(s.w, m));
    reinterpret_cast<float4*>(params)[i] = w;
    if (shadow != nullptr) {
      uint2 o;
      o.x = pack_bf16x2(w.x, w.y);
      o.y = pack_bf16x2(w.z, w.w);
      *reinterpret_cast<uint2*>(shadow + 4 * (size_t)i) = o;
    }
  }
}

}  // namespace dm

extern "C" {

int dm_gossip_stats_bytes() { return (int)sizeof(dm::GossipStats); }

// gs_apply: the half step h = params - fp32(lr(s)) * grads into send[s % 2] (`send`: 2 x numel fp32), s = the epoch word
// of my block (ctrl[rank]), with the block's learning-rate schedule.  `params` is only read.
int dm_gossip_apply(void* const* ctrl, int rank, const void* params, const void* grads, void* send, long long numel,
                    double lr0, double decay_rate, int decay_steps, int ctas, void* stream_) {
  using namespace dm;
  if (rank < 0 || rank >= SYNC_MAX_RANKS || (numel & 3) || numel / 4 > 0x7fffffffLL / 2 || send == nullptr) return -1;
  SyncArgs a;
  a.rank = rank; a.nranks = 1; a.k = 1; a.numel4 = (int)(numel / 4);
  a.lr0 = lr0; a.decay_rate = decay_rate; a.decay_steps = decay_steps;
  a.drop_keep = 0.f; a.drop_seed = 0; a.timeout_ns = 0;
  a.shadow = nullptr; a.mc_grads = nullptr; a.mc_params = nullptr;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (ctas < 1 || ctas > num_sms()) ctas = num_sms();
  return (int)launch_kernel(gs_apply_kernel, dim3(ctas), dim3(GS_THREADS), 0, st, a, reinterpret_cast<SyncCtrl*>(ctrl[rank]),
                            reinterpret_cast<const float*>(grads), reinterpret_cast<const float*>(params),
                            reinterpret_cast<float*>(send));
}

// The exchange of one iteration, after dm_gossip_apply: gs_barrier (the step is closed, the ring neighbours' barrier)
// and gs_mix (params and the bf16 shadow, null: none := the mean of the neighbourhood's half steps).  `ctrl` and `send`
// are the tables of every replica's control block and send buffers; `stats` dm_gossip_stats_bytes() bytes.  A wait past
// `timeout_ms` sets the error word.
int dm_gossip_exchange(void* const* ctrl, void* const* send, void* params, void* shadow_bf16, void* stats, int rank,
                       int nranks, long long numel, double timeout_ms, int ctas, void* stream_) {
  using namespace dm;
  if (nranks < 1 || nranks > SYNC_MAX_RANKS || rank < 0 || rank >= nranks || (numel & 3) ||
      numel / 4 > 0x7fffffffLL / 2 || stats == nullptr)
    return -1;
  GossipPeers P;
  for (int i = 0; i < SYNC_MAX_RANKS; ++i) {
    const int j = i < nranks ? i : rank;
    P.ctrl[i] = reinterpret_cast<SyncCtrl*>(ctrl[j]);
    P.send[i] = reinterpret_cast<const float*>(send[j]);
  }
  const unsigned long long tns = (unsigned long long)(timeout_ms * 1e6);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (ctas < 1 || ctas > num_sms()) ctas = num_sms();
  cudaError_t e = launch_kernel(gs_barrier_kernel, dim3(1), dim3(32), 0, st, P, reinterpret_cast<GossipStats*>(stats),
                                rank, nranks, tns);
  if (e != cudaSuccess) return (int)e;
  return (int)launch_kernel(gs_mix_kernel, dim3(ctas), dim3(GS_THREADS), 0, st, P, (const SyncCtrl*)P.ctrl[rank], rank,
                            nranks, (int)(numel / 4), reinterpret_cast<float*>(params),
                            reinterpret_cast<__nv_bfloat16*>(shadow_bf16));
}

}  // extern "C"
