// Forward-only evaluation head of the in-training validation pass (engine_cuda.CudaLeNetEngine.enqueue_eval).
//
//   eval_stamp   1 thread: opens a pass -- clears the running sums and stamps %globaltimer (start of the pass)
//   eval_head    CTA = ONE row, 128 threads x 4 hidden units: sum of the fc1 split-K partials, bias, ReLU (no dropout),
//                fc2, log-softmax cross entropy, first-maximum argmax.  The arithmetic is fc2_fwd_bwd's with train = 0
//                (csrc/lenet_simt.cu), so the logits are bit-identical to forward_logits(train=False).
//
// Unlike fc2_fwd_bwd, every piece of state is owned by the caller (EvalState + per-row workspace): the pass can sit in the
// training stream between two steps without touching the step's own workspaces.  Per chunk of rows, the last CTA
// (arrive_last_cta) adds the rows' loss terms in row order into a double and counts the correct rows as an integer; the
// chunks of a pass run one after the other on one stream and are folded into the running sums in chunk order, so a pass's
// record does not depend on CTA scheduling.  The last chunk's last CTA writes the record straight into page-locked host
// memory, like publish_status (csrc/fused_sync.cuh): the host reads it after an event that follows the pass.
#include "common.cuh"
#include "eval_state.cuh"
#include "host_utils.h"

namespace dm {

constexpr int EV_HID = 512;
constexpr int EV_NCLS = 10;
constexpr int EV_THREADS = EV_HID / 4;
constexpr int EV_MAX_SPLITS = 8;
constexpr int EV_MAX_ROWS = 4096;          // rows per chunk (the per-row workspace holds this many)
constexpr int EV_RECORD_WORDS = 8;         // u64 words per host record

// Per-row workspace: loss terms [EV_MAX_ROWS] fp32, then hit flags [EV_MAX_ROWS] u32.
struct EvalArgs {
  const float* h_part;             // [splits][rows,512] fc1 split-K partial accumulators (no bias)
  long long part_stride;
  int splits;
  const float* b1;                 // [512]
  const float* w2;                 // [512][10]
  const float* b2;                 // [10]
  const long long* labels;         // [rows]
  float* row_loss;                 // [EV_MAX_ROWS]
  unsigned int* row_hit;           // [EV_MAX_ROWS]
  EvalState* st;
  const uint32_t* step_ptr;        // device epoch word (global step of the weights), may be null
  const int32_t* status_ptr;       // snapshot outcome of the pass (csrc/eval_snapshot.cu: attempts, -1 = none), may be null
  unsigned long long* host_ring;   // [slots][EV_RECORD_WORDS] page-locked host memory, null: do not publish
  int ring_slots;
  float* logits_out;               // optional [rows,10]
  int last;                        // this chunk closes the pass
};

__global__ void eval_stamp_kernel(EvalState* st) {
  st->loss_sum = 0.0;
  st->correct = 0u;
  st->examples = 0u;
  st->t_begin = globaltimer_ns();
}

__global__ void __launch_bounds__(EV_THREADS) eval_head_kernel(EvalArgs a) {
  __shared__ float s_part[EV_THREADS / 32][12];
  __shared__ double s_loss[EV_THREADS];
  __shared__ unsigned int s_hit[EV_THREADS];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int row = blockIdx.x;
  float wf[4 * EV_NCLS];
  {
    const float4* wp = reinterpret_cast<const float4*>(a.w2) + 10 * t;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const float4 v = __ldg(wp + i);
      wf[4 * i] = v.x; wf[4 * i + 1] = v.y; wf[4 * i + 2] = v.z; wf[4 * i + 3] = v.w;
    }
  }
  const float4 b1v = __ldg(reinterpret_cast<const float4*>(a.b1) + t);
  const float b2v = lane < EV_NCLS ? __ldg(a.b2 + lane) : 0.f;
  pdl_wait();
  const int label = (int)a.labels[row];
  float4 part[EV_MAX_SPLITS];
#pragma unroll
  for (int s = 0; s < EV_MAX_SPLITS; ++s)
    part[s] = s < a.splits ? *(reinterpret_cast<const float4*>(a.h_part + (size_t)s * a.part_stride + (size_t)row * EV_HID) + t)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
  float hp[4] = {b1v.x, b1v.y, b1v.z, b1v.w};
#pragma unroll
  for (int s = 0; s < EV_MAX_SPLITS; ++s) { hp[0] += part[s].x; hp[1] += part[s].y; hp[2] += part[s].z; hp[3] += part[s].w; }
  float acc[EV_NCLS];
#pragma unroll
  for (int c = 0; c < EV_NCLS; ++c) acc[c] = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float h = hp[i] > 0.f ? hp[i] : 0.f;
#pragma unroll
    for (int c = 0; c < EV_NCLS; ++c) acc[c] = fmaf(h, wf[i * EV_NCLS + c], acc[c]);
  }
#pragma unroll
  for (int c = 0; c < EV_NCLS; ++c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
    if (lane == c) s_part[warp][c] = acc[c];
  }
  __syncthreads();
  if (warp == 0) {
    float logit = -INFINITY;
    if (lane < EV_NCLS) {
      logit = b2v;
#pragma unroll
      for (int w = 0; w < EV_THREADS / 32; ++w) logit += s_part[w][lane];
    }
    float m = logit;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    m = __shfl_sync(0xffffffffu, m, 0);
    const float e = lane < EV_NCLS ? __expf(logit - m) : 0.f;
    float ssum = e;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) ssum += __shfl_xor_sync(0xffffffffu, ssum, o);
    ssum = __shfl_sync(0xffffffffu, ssum, 0);
    // first index attaining the maximum (ties: lowest class, like the reference's in_top_k / argmax)
    const unsigned hit = __ballot_sync(0xffffffffu, lane < EV_NCLS && logit == m);
    const float l_label = __shfl_sync(0xffffffffu, logit, label);
    if (lane == 0) {
      a.row_loss[row] = __logf(ssum) - (l_label - m);
      a.row_hit[row] = (__ffs(hit) - 1) == label ? 1u : 0u;
    }
    if (a.logits_out && lane < EV_NCLS) a.logits_out[(size_t)row * EV_NCLS + lane] = logit;
  }
  __shared__ unsigned int s_last;
  if (!arrive_last_cta(&a.st->ticket, gridDim.x, 1, EV_THREADS, &s_last)) return;
  // last CTA: thread t adds rows [t * per, (t + 1) * per) in row order, thread 0 then adds the 128 partials in thread order
  const int rows = (int)gridDim.x;
  const int per = (rows + EV_THREADS - 1) / EV_THREADS;
  double l = 0.0;
  unsigned int h = 0u;
  for (int r = t * per; r < min(rows, (t + 1) * per); ++r) {
    l += (double)__ldcg(a.row_loss + r);
    h += __ldcg(a.row_hit + r);
  }
  s_loss[t] = l;
  s_hit[t] = h;
  __syncthreads();
  if (t != 0) return;
  double ls = 0.0;
  unsigned int hs = 0u;
  for (int i = 0; i < EV_THREADS; ++i) { ls += s_loss[i]; hs += s_hit[i]; }
  EvalState* st = a.st;
  st->loss_sum += ls;
  st->correct += hs;
  st->examples += (unsigned int)rows;
  if (!a.last || a.host_ring == nullptr) return;
  const unsigned long long t_end = globaltimer_ns();
  const unsigned int seq = st->seq + 1u;
  st->seq = seq;
  volatile unsigned long long* rec = a.host_ring + (size_t)EV_RECORD_WORDS * (seq % (unsigned)a.ring_slots);
  // seq word last, and cleared first: a reader that sees the same non-zero seq before and after reading the other words
  // has read one complete record
  rec[0] = 0ull;
  __threadfence_system();
  rec[1] = a.step_ptr ? (unsigned long long)*a.step_ptr : 0ull;
  rec[2] = st->t_begin;
  rec[3] = t_end;
  rec[4] = st->examples;
  rec[5] = st->correct;
  rec[6] = (unsigned long long)__double_as_longlong(st->loss_sum);
  rec[7] = a.status_ptr ? (unsigned long long)(long long)*a.status_ptr : 0ull;
  __threadfence_system();
  rec[0] = seq;
}

}  // namespace dm

extern "C" {

int dm_eval_state_bytes() { return (int)sizeof(dm::EvalState); }
int dm_eval_max_rows() { return dm::EV_MAX_ROWS; }

int dm_eval_stamp(void* state, void* stream) {
  dm::eval_stamp_kernel<<<1, 1, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<dm::EvalState*>(state));
  return (int)cudaGetLastError();
}

// One chunk of `rows` rows.  row_ws: [EV_MAX_ROWS] fp32 + [EV_MAX_ROWS] u32; state: EvalState opened by dm_eval_stamp.
// last != 0: the chunk closes the pass and publishes its record into host_ring (if not null).  status_ptr (may be null) is
// reported in the record's last word: the attempt that produced the pass's weight snapshot, -1 if none was consistent.
int dm_eval_head(const void* h_part, long long part_stride, int splits, const void* b1, const void* w2, const void* b2,
                 const void* labels, void* row_ws, void* state, const void* step_ptr, const void* status_ptr,
                 void* host_ring, int ring_slots, void* logits_out, int rows, int last, void* stream) {
  if (splits < 1 || splits > dm::EV_MAX_SPLITS || rows < 1 || rows > dm::EV_MAX_ROWS) return -1;
  if (host_ring != nullptr && ring_slots < 1) return -1;
  dm::EvalArgs a;
  a.h_part = reinterpret_cast<const float*>(h_part);
  a.part_stride = part_stride;
  a.splits = splits;
  a.b1 = reinterpret_cast<const float*>(b1);
  a.w2 = reinterpret_cast<const float*>(w2);
  a.b2 = reinterpret_cast<const float*>(b2);
  a.labels = reinterpret_cast<const long long*>(labels);
  a.row_loss = reinterpret_cast<float*>(row_ws);
  a.row_hit = reinterpret_cast<unsigned int*>(reinterpret_cast<float*>(row_ws) + dm::EV_MAX_ROWS);
  a.st = reinterpret_cast<dm::EvalState*>(state);
  a.step_ptr = reinterpret_cast<const uint32_t*>(step_ptr);
  a.status_ptr = reinterpret_cast<const int32_t*>(status_ptr);
  a.host_ring = reinterpret_cast<unsigned long long*>(host_ring);
  a.ring_slots = ring_slots;
  a.logits_out = reinterpret_cast<float*>(logits_out);
  a.last = last;
  return (int)dm::launch_kernel(dm::eval_head_kernel, dim3(rows), dim3(dm::EV_THREADS), 0,
                                reinterpret_cast<cudaStream_t>(stream), a);
}

}  // extern "C"
