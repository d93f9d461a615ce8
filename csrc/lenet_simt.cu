// SIMT kernels of the LeNet pipeline: fc2 and the loss, whose GEMM view is too thin for tensor cores
// (SURVEY §2.4 K8: N = 10), fused with the fc1 epilogue and the loss bookkeeping.
//
//   fc2_fwd_bwd    K6 epilogue (bias+ReLU+dropout on the fc1 split-K partials, K7) + K8 + K9 + K10 and
//                  their backward: dlogits, d(fc1 pre-activation)   (src/mnist.py:136-145,149-164)
//   fc2_wgrad      fc2 weight/bias gradients and the fc1 bias gradient
#include "common.cuh"
#include "host_utils.h"

namespace dm {

// =====================================================================================================
// fc2 + softmax cross entropy + accuracy, forward and backward, as two kernels:
//
//   fc2_fwd_bwd   (critical path)  CTA = ONE batch row, 128 threads x 4 hidden units.  fc1 epilogue (sum of the
//                 split-K partials, bias, ReLU, dropout), fc2, softmax, loss/accuracy, dlogits and
//                 d(fc1 pre-activation).  Every global load of a thread is independent of every other, so a
//                 CTA pays ONE memory round trip; B CTAs are all resident at once.
//   fc2_wgrad     (side branch of the step graph, consumed only by the aggregation kernel)
//                 fc2 weight/bias gradients and the fc1 bias gradient from the activations / dlogits the first
//                 kernel saved.  CTA = 8 hidden units x all rows, staged through shared memory; plain stores
//                 (no atomics, nothing to pre-zero).
// =====================================================================================================
constexpr int HID = 512;
constexpr int NCLS = 10;
constexpr int DL_LD = 12;          // dlogits row stride (floats): 48 B rows -> 16-byte vector loads
constexpr int F2_THREADS = HID / 4;
constexpr int F2_MAX_SPLITS = 8;

struct Fc2Args {
  const float* h_part;       // [splits][B,512] fc1 split-K partial accumulators (no bias)
  long long part_stride;     // elements between partials
  int splits;
  const float* b1;           // [512]
  const float* w2;           // [512][10]
  const float* b2;           // [10]
  const long long* labels;   // [B]
  __nv_bfloat16* dh;         // [B,512] out: d loss / d fc1 pre-activation                      (train)
  float* h_out;              // [B,512] out: post ReLU/dropout activations (fc2_wgrad operand)  (train)
  float* dl_out;             // [B,12]  out: d loss / d logits, columns 10-11 zero              (train)
  float* loss_acc;           // [2]: sum of per-row loss / B, number of correct / B  (pre-zeroed)
  float2* row_terms;         // [B] per-row (loss, hit) terms; null: g_f2_row_terms, added up by the launch's last CTA
  float* logits_out;         // optional [B,10]
  int B;
  int train;
  uint32_t seed_mix;         // dropout_seed_mix(seed, 0, rank); the step is added on the device
  const uint32_t* step_ptr;  // device-resident step counter (CUDA-graph friendly), may be null
  float keep_prob;
  float inv_batch;           // 1 / (rows that make up the mean)
};

// Per-row (loss, hit) terms, added up in row order by fc2_loss_sum: the reported loss and accuracy do not depend on the
// order in which the rows' CTAs finish.  dm_fc2_fwd_bwd stores them into a static workspace and its last CTA
// (arrive_last_cta) adds them; dm_fc2_fwd_bwd_rows stores them into the caller's buffer and exits, and
// dm_fc2_loss_sum adds them later, where nothing on the training step's data-gradient chain waits for the sum.
constexpr int F2_MAX_ROWS = 1 << 16;                      // batch limit of dm_fc2_fwd_bwd
// One launch of dm_fc2_fwd_bwd in flight per device: the workspace and ticket are static (see arrive_last_cta).
__device__ float2 g_f2_row_terms[F2_MAX_ROWS];
__device__ unsigned int g_f2_ticket;

int fc2_fwd_bwd_max_batch() { return F2_MAX_ROWS; }

// One warp: lane l adds rows l, l + 32, ... in row order (16 rows' loads in flight per round: one L2 round trip at
// B <= 512), then a fixed butterfly; lane 0 adds the two sums onto the pre-zeroed loss words.
DMNIST_DEVICE void fc2_loss_sum(const float2* terms, int rows, float* loss_acc) {
  const int lane = threadIdx.x & 31;
  float l = 0.f, h = 0.f;
  for (int r0 = lane; r0 < rows; r0 += 32 * 16) {
    float2 v[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) v[u] = r0 + 32 * u < rows ? __ldcg(terms + r0 + 32 * u) : make_float2(0.f, 0.f);
#pragma unroll
    for (int u = 0; u < 16; ++u)
      if (r0 + 32 * u < rows) { l += v[u].x; h += v[u].y; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l += __shfl_xor_sync(0xffffffffu, l, o);
    h += __shfl_xor_sync(0xffffffffu, h, o);
  }
  if (lane == 0) {
    // fire-and-forget: the warp does not wait for a load of the words (same rounding as +=)
    atomicAdd(loss_acc, l);
    atomicAdd(loss_acc + 1, h);
  }
}

__global__ void __launch_bounds__(32) fc2_loss_sum_kernel(const float2* terms, int rows, float* loss_acc) {
  pdl_wait();
  fc2_loss_sum(terms, rows, loss_acc);
}

__global__ void __launch_bounds__(F2_THREADS) fc2_fwd_bwd_kernel(Fc2Args a) {
  __shared__ float s_part[F2_THREADS / 32][DL_LD];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int row = blockIdx.x;
  // parameters first: they were final before the previous kernel even started, so these loads overlap its tail
  float wf[4 * NCLS];                                  // w2 rows 4t .. 4t+3: 40 consecutive floats
  {
    const float4* wp = reinterpret_cast<const float4*>(a.w2) + 10 * t;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const float4 v = __ldg(wp + i);
      wf[4 * i] = v.x; wf[4 * i + 1] = v.y; wf[4 * i + 2] = v.z; wf[4 * i + 3] = v.w;
    }
  }
  const float4 b1v = __ldg(reinterpret_cast<const float4*>(a.b1) + t);
  const float b2v = lane < NCLS ? __ldg(a.b2 + lane) : 0.f;
  pdl_wait();
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)
  const uint32_t step = a.step_ptr ? *a.step_ptr : 0u;
  const int label = (int)a.labels[row];
  float4 part[F2_MAX_SPLITS];
#pragma unroll
  for (int s = 0; s < F2_MAX_SPLITS; ++s)
    part[s] = s < a.splits ? *(reinterpret_cast<const float4*>(a.h_part + (size_t)s * a.part_stride + (size_t)row * HID) + t)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
  float hp[4] = {b1v.x, b1v.y, b1v.z, b1v.w};
#pragma unroll
  for (int s = 0; s < F2_MAX_SPLITS; ++s) { hp[0] += part[s].x; hp[1] += part[s].y; hp[2] += part[s].z; hp[3] += part[s].w; }

  const uint32_t mix = a.seed_mix + step * 0x9E3779B9u;
  const uint32_t thresh = (uint32_t)(a.keep_prob * 16777216.f);
  const float inv_keep = a.train ? 1.f / a.keep_prob : 1.f;
  float h[4], acc[NCLS];
#pragma unroll
  for (int c = 0; c < NCLS; ++c) acc[c] = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    bool on = hp[i] > 0.f;
    if (a.train) on = on && dropout_keep(mix, (uint32_t)(row * HID + 4 * t + i), thresh);
    h[i] = on ? hp[i] * inv_keep : 0.f;
#pragma unroll
    for (int c = 0; c < NCLS; ++c) acc[c] = fmaf(h[i], wf[i * NCLS + c], acc[c]);
  }
#pragma unroll
  for (int c = 0; c < NCLS; ++c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
    if (lane == c) s_part[warp][c] = acc[c];
  }
  __syncthreads();
  // every warp finishes the row redundantly (lane c owns class c): no second barrier, no broadcast through memory
  float logit = -INFINITY;
  if (lane < NCLS) {
    logit = b2v;
#pragma unroll
    for (int w = 0; w < F2_THREADS / 32; ++w) logit += s_part[w][lane];
  }
  float m = logit;
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));     // lanes 0-15 hold the 10 classes
  m = __shfl_sync(0xffffffffu, m, 0);
  const float e = lane < NCLS ? __expf(logit - m) : 0.f;
  float ssum = e;
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) ssum += __shfl_xor_sync(0xffffffffu, ssum, o);
  ssum = __shfl_sync(0xffffffffu, ssum, 0);
  const float dl_mine = lane < NCLS ? (e / ssum - (lane == label ? 1.f : 0.f)) * a.inv_batch : 0.f;
  if (warp == 0) {
    // first index attaining the maximum (ties: lowest class, like the reference's in_top_k / argmax)
    const unsigned hit = __ballot_sync(0xffffffffu, lane < NCLS && logit == m);
    const float l_label = __shfl_sync(0xffffffffu, logit, label);
    if (lane == 0)
      (a.row_terms ? a.row_terms : g_f2_row_terms)[row] =
          make_float2((__logf(ssum) - (l_label - m)) * a.inv_batch, ((__ffs(hit) - 1) == label ? 1.f : 0.f) * a.inv_batch);
    if (a.logits_out && lane < NCLS) a.logits_out[(size_t)row * NCLS + lane] = logit;
    if (a.train && lane < DL_LD) a.dl_out[(size_t)row * DL_LD + lane] = dl_mine;
  }
  if (!a.row_terms) {
    __shared__ unsigned int s_last;
    if (arrive_last_cta(&g_f2_ticket, gridDim.x, 1, F2_THREADS, &s_last) && warp == 0)
      fc2_loss_sum(g_f2_row_terms, (int)gridDim.x, a.loss_acc);
  }
  if (!a.train) return;
  float d[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int c = 0; c < NCLS; ++c) {
    const float dl = __shfl_sync(0xffffffffu, dl_mine, c);
#pragma unroll
    for (int i = 0; i < 4; ++i) d[i] = fmaf(dl, wf[i * NCLS + c], d[i]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) d[i] = (h[i] != 0.f) ? d[i] * inv_keep : 0.f;   // ReLU and dropout masks: h == 0 exactly where either killed it
  const size_t o = (size_t)row * HID + 4 * t;
  *reinterpret_cast<uint2*>(a.dh + o) = make_uint2(pack_bf16x2(d[0], d[1]), pack_bf16x2(d[2], d[3]));
  *reinterpret_cast<float4*>(a.h_out + o) = make_float4(h[0], h[1], h[2], h[3]);
}

// fc2 weight / bias gradients and the fc1 bias gradient.  grid = 512 / 8 CTAs of 256 threads.
//   output o < 80       : g_w2[j0 + o / 10][o % 10] = sum_r h[r][j] * dl[r][c]
//   output 80 .. 87     : g_b1[j0 + o - 80]         = sum_r dh[r][j]
//   output 88 .. 97     : g_b2[o - 88]              = sum_r dl[r][c]        (CTA 0 only)
// DECAY (--weight_decay): each output is fma(decay, v, sum) with one rounding, v = w2 / b1 / b2, and each CTA stores the
// sum of the squares of the variables it owns, in double and a fixed order, into decay_part[blockIdx.x].
constexpr int FW_J = 8;
constexpr int FW_ROWS = 256;
struct Fc2Decay {
  const float* w2;           // [512][10]
  const float* b2;           // [10]
  const float* b1;           // [512]
  float decay;
  double* part;              // [512 / FW_J]
};
template <bool DECAY>
__global__ void __launch_bounds__(256) fc2_wgrad_kernel(const float* __restrict__ h,            // [B,512]
                                                        const float* __restrict__ dl,           // [B,12]
                                                        const __nv_bfloat16* __restrict__ dh,   // [B,512]
                                                        float* __restrict__ g_w2, float* __restrict__ g_b2,
                                                        float* __restrict__ g_b1, int B, Fc2Decay dk) {
  __shared__ __align__(16) float s_h[FW_ROWS][FW_J];
  __shared__ __align__(16) float s_dh[FW_ROWS][FW_J];
  __shared__ __align__(16) float s_dl[FW_ROWS][DL_LD];
  __shared__ float s_red[128];
  pdl_wait();
  const int t = threadIdx.x, j0 = blockIdx.x * FW_J;
  const int o = t & 127, half = t >> 7;
  const int kind = o < 80 ? 0 : (o < 88 ? 1 : (o < 98 ? 2 : 3));
  const int oj = kind == 0 ? o / NCLS : (kind == 1 ? o - 80 : 0);
  const int oc = kind == 0 ? o % NCLS : (kind == 2 ? o - 88 : 0);
  float acc = 0.f;
  for (int r0 = 0; r0 < B; r0 += FW_ROWS) {
    const int rows = min(FW_ROWS, B - r0);
    __syncthreads();
    if (t < rows) {
      const size_t src = (size_t)(r0 + t) * HID + j0;
      const float4 h0 = *reinterpret_cast<const float4*>(h + src), h1 = *reinterpret_cast<const float4*>(h + src + 4);
      const uint4 dv = *reinterpret_cast<const uint4*>(dh + src);
      const float4* dlp = reinterpret_cast<const float4*>(dl + (size_t)(r0 + t) * DL_LD);
      const float4 l0 = dlp[0], l1 = dlp[1], l2 = dlp[2];
      *reinterpret_cast<float4*>(&s_h[t][0]) = h0;
      *reinterpret_cast<float4*>(&s_h[t][4]) = h1;
      const uint32_t d32[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        s_dh[t][2 * i] = __uint_as_float(d32[i] << 16);
        s_dh[t][2 * i + 1] = __uint_as_float(d32[i] & 0xffff0000u);
      }
      *reinterpret_cast<float4*>(&s_dl[t][0]) = l0;
      *reinterpret_cast<float4*>(&s_dl[t][4]) = l1;
      *reinterpret_cast<float4*>(&s_dl[t][8]) = l2;
    }
    __syncthreads();
    if (kind == 0) {
#pragma unroll 8
      for (int r = half; r < rows; r += 2) acc = fmaf(s_h[r][oj], s_dl[r][oc], acc);
    } else if (kind == 1) {
#pragma unroll 8
      for (int r = half; r < rows; r += 2) acc += s_dh[r][oj];
    } else if (kind == 2) {
#pragma unroll 8
      for (int r = half; r < rows; r += 2) acc += s_dl[r][oc];
    }
  }
  if (half == 1) s_red[o] = acc;
  __syncthreads();
  if (half == 0) {
    acc += s_red[o];
    if (DECAY) {
      float v = 0.f;                               // outputs this CTA does not store decay nothing
      if (kind == 0) v = dk.w2[(j0 + oj) * NCLS + oc];
      else if (kind == 1) v = dk.b1[j0 + oj];
      else if (kind == 2 && blockIdx.x == 0) v = dk.b2[oc];
      acc = fma_rn(dk.decay, v, acc);
      s_red[o] = v;                                // (every thread has read s_red above; this is its own slot)
    }
    if (kind == 0) g_w2[(size_t)(j0 + oj) * NCLS + oc] = acc;
    else if (kind == 1) g_b1[j0 + oj] = acc;
    else if (kind == 2 && blockIdx.x == 0) g_b2[oc] = acc;
  }
  if (DECAY) {
    __syncthreads();
    if (t < 32) {
      // lane l: outputs l, l + 32, l + 64, l + 96 in order, then a fixed butterfly
      double s = 0.0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const double v = s_red[t + 32 * i];
        s += v * v;                                // the square of a float is exact in double
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
      if (t == 0) dk.part[blockIdx.x] = s;
    }
  }
}

template <bool DECAY>
int launch_fc2_wgrad(const void* scratch_h, const void* scratch_dl, const void* dh, void* g_w2, void* g_b2, void* g_b1,
                            int B, Fc2Decay dk, void* stream) {
  // side-branch kernel: it has to share SMs with the tensor-core kernels (max-shared L1 split), see dm_fused_sync_bucket
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(fc2_wgrad_kernel<DECAY>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                    cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  return (int)launch_kernel(fc2_wgrad_kernel<DECAY>, dim3(HID / FW_J), dim3(256), 0,
                                reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const float*>(scratch_h),
                                reinterpret_cast<const float*>(scratch_dl), reinterpret_cast<const __nv_bfloat16*>(dh),
                                reinterpret_cast<float*>(g_w2), reinterpret_cast<float*>(g_b2),
                                reinterpret_cast<float*>(g_b1), B, dk);
}

// row_terms == nullptr: the per-row terms go to g_f2_row_terms and the launch's last CTA adds them onto loss_acc
int launch_fc2_fwd_bwd(const void* h_part, long long part_stride, int splits, const void* b1, const void* w2,
                       const void* b2, const void* labels, void* dh, void* scratch_h, void* scratch_dl, void* loss_acc,
                       void* row_terms, void* logits_out, int B, int train, unsigned int seed_mix, const void* step_ptr,
                       float keep_prob, void* stream) {
  if (splits < 1 || splits > F2_MAX_SPLITS || B < 1 || B > F2_MAX_ROWS) return -1;
  Fc2Args a;
  a.h_part = reinterpret_cast<const float*>(h_part);
  a.part_stride = part_stride;
  a.splits = splits;
  a.b1 = reinterpret_cast<const float*>(b1);
  a.w2 = reinterpret_cast<const float*>(w2);
  a.b2 = reinterpret_cast<const float*>(b2);
  a.labels = reinterpret_cast<const long long*>(labels);
  a.dh = reinterpret_cast<__nv_bfloat16*>(dh);
  a.h_out = reinterpret_cast<float*>(scratch_h);
  a.dl_out = reinterpret_cast<float*>(scratch_dl);
  a.loss_acc = reinterpret_cast<float*>(loss_acc);
  a.row_terms = reinterpret_cast<float2*>(row_terms);
  a.logits_out = reinterpret_cast<float*>(logits_out);
  a.B = B; a.train = train; a.seed_mix = seed_mix;
  a.step_ptr = reinterpret_cast<const uint32_t*>(step_ptr);
  a.keep_prob = keep_prob;
  a.inv_batch = 1.f / (float)B;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(fc2_fwd_bwd_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  return (int)launch_kernel(fc2_fwd_bwd_kernel, dim3(B), dim3(F2_THREADS), 0, reinterpret_cast<cudaStream_t>(stream), a);
}

}  // namespace dm

extern "C" {

// Critical-path half: logits / loss / accuracy and (train) dh, h_out, dl_out.  scratch_h [B,512] fp32 and
// scratch_dl [B,12] fp32 are only touched when train != 0.
int dm_fc2_fwd_bwd(const void* h_part, long long part_stride, int splits, const void* b1, const void* w2, const void* b2,
                   const void* labels, void* dh, void* scratch_h, void* scratch_dl, void* loss_acc, void* logits_out,
                   int B, int train, unsigned int seed_mix, const void* step_ptr, float keep_prob, void* stream) {
  return dm::launch_fc2_fwd_bwd(h_part, part_stride, splits, b1, w2, b2, labels, dh, scratch_h, scratch_dl, loss_acc,
                                nullptr, logits_out, B, train, seed_mix, step_ptr, keep_prob, stream);
}

// The same, except that the per-row (loss, hit) terms go to row_terms ([B] float pairs) and loss_acc is not touched:
// dm_fc2_loss_sum(row_terms, B, loss_acc) then adds them as dm_fc2_fwd_bwd would have, to the bit.  The training step
// runs the sum on a side branch, so nothing on its data-gradient chain waits for it.
int dm_fc2_fwd_bwd_rows(const void* h_part, long long part_stride, int splits, const void* b1, const void* w2,
                        const void* b2, const void* labels, void* dh, void* scratch_h, void* scratch_dl, void* row_terms,
                        void* logits_out, int B, int train, unsigned int seed_mix, const void* step_ptr, float keep_prob,
                        void* stream) {
  if (row_terms == nullptr) return -1;
  return dm::launch_fc2_fwd_bwd(h_part, part_stride, splits, b1, w2, b2, labels, dh, scratch_h, scratch_dl, nullptr,
                                row_terms, logits_out, B, train, seed_mix, step_ptr, keep_prob, stream);
}

// loss_acc[0] += the rows' loss terms, loss_acc[1] += their hit terms, each in row order (one warp).
int dm_fc2_loss_sum(const void* row_terms, int B, void* loss_acc, void* stream) {
  if (row_terms == nullptr || loss_acc == nullptr || B < 1) return -1;
  return (int)dm::launch_kernel(dm::fc2_loss_sum_kernel, dim3(1), dim3(32), 0, reinterpret_cast<cudaStream_t>(stream),
                                reinterpret_cast<const float2*>(row_terms), B, reinterpret_cast<float*>(loss_acc));
}

// Side-branch half: g_w2 [512][10], g_b2 [10], g_b1 [512] (plain stores).
int dm_fc2_wgrad(const void* scratch_h, const void* scratch_dl, const void* dh, void* g_w2, void* g_b2, void* g_b1, int B,
                 void* stream) {
  return dm::launch_fc2_wgrad<false>(scratch_h, scratch_dl, dh, g_w2, g_b2, g_b1, B, dm::Fc2Decay{}, stream);
}

// The same with L2 decay: g_w2 / g_b2 / g_b1 gain decay * w2 / b2 / b1 (one rounding each); decay_part receives
// dm_fc2_wgrad_decay_ctas() doubles, the squares of the variables each CTA owns, summed.
int dm_fc2_wgrad_decay_ctas() { return dm::HID / dm::FW_J; }

int dm_fc2_wgrad_decay(const void* scratch_h, const void* scratch_dl, const void* dh, void* g_w2, void* g_b2, void* g_b1,
                       int B, const void* w2, const void* b2, const void* b1, float decay, void* decay_part, void* stream) {
  if (w2 == nullptr || b2 == nullptr || b1 == nullptr || decay_part == nullptr) return -1;
  const dm::Fc2Decay dk{reinterpret_cast<const float*>(w2), reinterpret_cast<const float*>(b2),
                        reinterpret_cast<const float*>(b1), decay, reinterpret_cast<double*>(decay_part)};
  return dm::launch_fc2_wgrad<true>(scratch_h, scratch_dl, dh, g_w2, g_b2, g_b1, B, dk, stream);
}

}  // extern "C"
