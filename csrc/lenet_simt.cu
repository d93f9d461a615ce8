// SIMT kernels of the LeNet pipeline: the ops whose GEMM view is too thin for tensor cores
// (SURVEY §2.4 K1: K = 25; K8: N = 10) plus the fused pooling / ReLU / loss bookkeeping.
//
//   conv1_fwd      K1+K2+K3+K4  conv5x5(1->32,SAME) + bias + ReLU + maxpool2x2   (src/mnist.py:107-118)
//   fc2_loss       K6 epilogue (bias+ReLU+dropout on the fc1 accumulator, K7) + K8 + K9 + K10 and
//                  their backward: dlogits, fc2 wgrad/bgrad, d(fc1 pre-activation), fc1 bgrad
//                  (src/mnist.py:136-145,149-164)
//   unpool2        backward of maxpool2 + ReLU2 (scatter to the argmax position) + conv2 bias grad
//   conv1_wgrad    backward of maxpool1 + ReLU1 fused with the conv1 weight/bias gradient
//
// Pooling stores one code byte per pooled element: bits 0-1 = argmax position (dy*2+dx),
// bit 2 = ReLU active; the backward kernels need nothing else.
#include "common.cuh"
#include "host_utils.h"

namespace dm {

// Two channels per call (the same rounding as one fmaf each): keeps the channel-pair register layout of the loops.
DMNIST_DEVICE float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}


// =====================================================================================================
// conv1 forward, fused.  One CTA per (image, pair of pooled rows): 2 x 14 pooled positions x 32 channels.
// Work item = (pooled position, group of 8 channels): 4 conv outputs x 8 channels x 25 taps = 800 FMA,
// fed from shared memory (12 input values + 10 weight vectors per filter row).
// =====================================================================================================
constexpr int C1_THREADS = 128;   // 112 work items + 16 idle lanes

struct ZeroRanges {
  float* ptr[3];
  int n[3];
};

__global__ void __launch_bounds__(C1_THREADS) conv1_fwd_kernel(const float* __restrict__ images,  // [B,28,28]
                                                               const float* __restrict__ w,       // [25][32]
                                                               const float* __restrict__ bias,    // [32]
                                                               __nv_bfloat16* __restrict__ out,   // [B,14,14,32]
                                                               uint8_t* __restrict__ code,        // [B,14,14,32]
                                                               ZeroRanges zr) {
  pdl_wait();
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)
  // First kernel of a training step: also clears the gradient regions that later kernels accumulate into
  // with atomics and the loss accumulator (replaces three memset nodes of the step graph).
  {
    const int gi = blockIdx.x * C1_THREADS + threadIdx.x;
#pragma unroll
    for (int r = 0; r < 3; ++r)
      if (zr.ptr[r] != nullptr)
        for (int i = gi; i < zr.n[r]; i += gridDim.x * C1_THREADS) zr.ptr[r][i] = 0.f;
  }
  __shared__ float s_img[8][32];        // input rows 4*u-2 .. 4*u+5, columns -2 .. 29 (zero halo)
  __shared__ __align__(16) float s_w[25][32];
  __shared__ float s_b[32];
  const int b = blockIdx.x / 7, u = blockIdx.x - b * 7;   // u: pooled rows 2u, 2u+1
  const int row0 = 4 * u - 2;
  for (int i = threadIdx.x; i < 8 * 32; i += C1_THREADS) {
    const int r = i >> 5, c = i & 31;
    const int y = row0 + r, x = c - 2;
    s_img[r][c] = (y >= 0 && y < 28 && x >= 0 && x < 28) ? __ldg(images + (size_t)b * 784 + y * 28 + x) : 0.f;
  }
  for (int i = threadIdx.x; i < 200; i += C1_THREADS)
    reinterpret_cast<float4*>(&s_w[0][0])[i] = __ldg(reinterpret_cast<const float4*>(w) + i);
  if (threadIdx.x < 32) s_b[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();

  const int cg = threadIdx.x & 3, pos = threadIdx.x >> 2;
  if (pos >= 28) return;
  const int pr = pos / 14, pc = pos - pr * 14;          // pooled row (local) / col
  // channel pairs: input value broadcast to both halves
  float2 acc2[4][4];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc2[p][j] = make_float2(0.f, 0.f);
#pragma unroll 1
  for (int kh = 0; kh < 5; ++kh) {
    float r0[6], r1[6];                                   // the two input rows this filter row touches
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      r0[c] = s_img[2 * pr + kh][2 * pc + c];
      r1[c] = s_img[2 * pr + kh + 1][2 * pc + c];
    }
#pragma unroll
    for (int kw = 0; kw < 5; ++kw) {
      const float4 w0 = *reinterpret_cast<const float4*>(&s_w[kh * 5 + kw][cg * 8]);
      const float4 w1 = *reinterpret_cast<const float4*>(&s_w[kh * 5 + kw][cg * 8 + 4]);
      const float2 wv[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y),
                            make_float2(w1.z, w1.w)};
      const float2 a00 = make_float2(r0[kw], r0[kw]), a01 = make_float2(r0[kw + 1], r0[kw + 1]);
      const float2 a10 = make_float2(r1[kw], r1[kw]), a11 = make_float2(r1[kw + 1], r1[kw + 1]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc2[0][j] = fma2_rn(a00, wv[j], acc2[0][j]);
        acc2[1][j] = fma2_rn(a01, wv[j], acc2[1][j]);
        acc2[2][j] = fma2_rn(a10, wv[j], acc2[2][j]);
        acc2[3][j] = fma2_rn(a11, wv[j], acc2[3][j]);
      }
    }
  }
  float acc[4][8];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[p][2 * j] = acc2[p][j].x; acc[p][2 * j + 1] = acc2[p][j].y; }
  uint32_t packed[4];
  uint32_t cd[2] = {0u, 0u};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float m = acc[0][j];
    uint32_t idx = 0;
#pragma unroll
    for (int p = 1; p < 4; ++p)
      if (acc[p][j] > m) { m = acc[p][j]; idx = p; }
    m += s_b[cg * 8 + j];
    const bool active = m > 0.f;
    cd[j >> 2] |= (idx | (active ? 4u : 0u)) << ((j & 3) * 8);
    const float o = active ? m : 0.f;
    if (j & 1) packed[j >> 1] = pack_bf16x2(__uint_as_float(packed[j >> 1]), o);
    else packed[j >> 1] = __float_as_uint(o);
  }
  const size_t o = (((size_t)b * 14 + 2 * u + pr) * 14 + pc) * 32 + cg * 8;
  *reinterpret_cast<uint4*>(out + o) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
  *reinterpret_cast<uint2*>(code + o) = make_uint2(cd[0], cd[1]);
}

// conv1 forward, second generation.  Same CTA = (image, pair of pooled rows), but a thread owns TWO horizontally adjacent
// pooled positions (2 x 4 conv outputs) x 8 channels: the ten 16-byte weight loads of a filter row now feed 160 packed
// FMAs instead of 80 and the input window is four aligned 16-byte loads, so the loop is bound by the FMA pipe rather
// than by shared-memory issue slots (the first version spent more instructions on loads and address arithmetic than
// on FMAs).  64 threads: 56 work items = 2 rows x 7 column pairs x 4 groups.
constexpr int C1B_THREADS = 64;

__global__ void __launch_bounds__(C1B_THREADS) conv1_fwd2_kernel(const float* __restrict__ images,  // [B,28,28]
                                                                 const float* __restrict__ w,       // [25][32]
                                                                 const float* __restrict__ bias,    // [32]
                                                                 __nv_bfloat16* __restrict__ out,   // [B,14,14,32]
                                                                 uint8_t* __restrict__ code,        // [B,14,14,32]
                                                                 ZeroRanges zr) {
  __shared__ __align__(16) float s_img[8][32];        // input rows 4*u-2 .. 4*u+5, columns -2 .. 29 (zero halo)
  __shared__ __align__(16) float s_w[25][32];
  __shared__ float s_b[32];
  const int b = blockIdx.x / 7, u = blockIdx.x - b * 7;   // u: pooled rows 2u, 2u+1
  // weights and bias are final long before the previous kernel of the stream started: fetch them ahead of the wait
  for (int i = threadIdx.x; i < 200; i += C1B_THREADS)
    reinterpret_cast<float4*>(&s_w[0][0])[i] = __ldg(reinterpret_cast<const float4*>(w) + i);
  if (threadIdx.x < 32) s_b[threadIdx.x] = __ldg(bias + threadIdx.x);
  pdl_wait();
  {
    const int gi = blockIdx.x * C1B_THREADS + threadIdx.x;
#pragma unroll
    for (int r = 0; r < 3; ++r)
      if (zr.ptr[r] != nullptr)
        for (int i = gi; i < zr.n[r]; i += gridDim.x * C1B_THREADS) zr.ptr[r][i] = 0.f;
  }
  const int row0 = 4 * u - 2;
  for (int i = threadIdx.x; i < 8 * 32; i += C1B_THREADS) {
    const int r = i >> 5, c = i & 31;
    const int y = row0 + r, x = c - 2;
    s_img[r][c] = (y >= 0 && y < 28 && x >= 0 && x < 28) ? __ldg(images + (size_t)b * 784 + y * 28 + x) : 0.f;
  }
  __syncthreads();

  const int cg = threadIdx.x & 3, item = threadIdx.x >> 2;
  if (item >= 14) return;
  const int pr = item / 7, pair = item - pr * 7;          // pooled row (local), pair of pooled columns
  float2 acc[8][4];                                       // [conv output: row * 4 + column][channel pair]
#pragma unroll
  for (int p = 0; p < 8; ++p)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[p][j] = make_float2(0.f, 0.f);
#pragma unroll 1
  for (int kh = 0; kh < 5; ++kh) {
    float r0[8], r1[8];                                   // the two input rows this filter row touches, 8 columns
    {
      const float4* p0 = reinterpret_cast<const float4*>(&s_img[2 * pr + kh][4 * pair]);
      const float4* p1 = reinterpret_cast<const float4*>(&s_img[2 * pr + kh + 1][4 * pair]);
      const float4 a = p0[0], bq = p0[1], c = p1[0], d = p1[1];
      r0[0] = a.x; r0[1] = a.y; r0[2] = a.z; r0[3] = a.w; r0[4] = bq.x; r0[5] = bq.y; r0[6] = bq.z; r0[7] = bq.w;
      r1[0] = c.x; r1[1] = c.y; r1[2] = c.z; r1[3] = c.w; r1[4] = d.x; r1[5] = d.y; r1[6] = d.z; r1[7] = d.w;
    }
#pragma unroll
    for (int kw = 0; kw < 5; ++kw) {
      const float4 w0 = *reinterpret_cast<const float4*>(&s_w[kh * 5 + kw][cg * 8]);
      const float4 w1 = *reinterpret_cast<const float4*>(&s_w[kh * 5 + kw][cg * 8 + 4]);
      const float2 wv[4] = {make_float2(w0.x, w0.y), make_float2(w0.z, w0.w), make_float2(w1.x, w1.y),
                            make_float2(w1.z, w1.w)};
#pragma unroll
      for (int col = 0; col < 4; ++col) {
        const float2 a0 = make_float2(r0[col + kw], r0[col + kw]), a1 = make_float2(r1[col + kw], r1[col + kw]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[col][j] = fma2_rn(a0, wv[j], acc[col][j]);
          acc[4 + col][j] = fma2_rn(a1, wv[j], acc[4 + col][j]);
        }
      }
    }
  }
#pragma unroll
  for (int pos = 0; pos < 2; ++pos) {
    uint32_t packed[4];
    uint32_t cd[2] = {0u, 0u};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // window order = argmax code: 0 (dy0,dx0), 1 (dy0,dx1), 2 (dy1,dx0), 3 (dy1,dx1)
      const float v[4] = {(j & 1) ? acc[2 * pos][j >> 1].y : acc[2 * pos][j >> 1].x,
                          (j & 1) ? acc[2 * pos + 1][j >> 1].y : acc[2 * pos + 1][j >> 1].x,
                          (j & 1) ? acc[4 + 2 * pos][j >> 1].y : acc[4 + 2 * pos][j >> 1].x,
                          (j & 1) ? acc[4 + 2 * pos + 1][j >> 1].y : acc[4 + 2 * pos + 1][j >> 1].x};
      float m = v[0];
      uint32_t idx = 0;
#pragma unroll
      for (int p = 1; p < 4; ++p)
        if (v[p] > m) { m = v[p]; idx = p; }
      m += s_b[cg * 8 + j];
      const bool active = m > 0.f;
      cd[j >> 2] |= (idx | (active ? 4u : 0u)) << ((j & 3) * 8);
      const float o = active ? m : 0.f;
      if (j & 1) packed[j >> 1] = pack_bf16x2(__uint_as_float(packed[j >> 1]), o);
      else packed[j >> 1] = __float_as_uint(o);
    }
    const size_t o = (((size_t)b * 14 + 2 * u + pr) * 14 + 2 * pair + pos) * 32 + cg * 8;
    *reinterpret_cast<uint4*>(out + o) = make_uint4(packed[0], packed[1], packed[2], packed[3]);
    *reinterpret_cast<uint2*>(code + o) = make_uint2(cd[0], cd[1]);
  }
}

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
  float* logits_out;         // optional [B,10]
  int B;
  int train;
  uint32_t seed_mix;         // dropout_seed_mix(seed, 0, rank); the step is added on the device
  const uint32_t* step_ptr;  // device-resident step counter (CUDA-graph friendly), may be null
  float keep_prob;
  float inv_batch;           // 1 / (rows that make up the mean)
};

// Per-row (loss, hit) terms, added up in row order by the last CTA (arrive_last_cta): the reported loss and accuracy do
// not depend on the order in which the rows' CTAs finish.
constexpr int F2_MAX_ROWS = 1 << 16;                      // batch limit of dm_fc2_fwd_bwd
// One launch of this kernel in flight per device: the workspace and ticket are static (see arrive_last_cta).
__device__ float g_f2_row_terms[F2_MAX_ROWS * 2];
__device__ unsigned int g_f2_ticket;

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
    if (lane == 0) {
      g_f2_row_terms[2 * row] = (__logf(ssum) - (l_label - m)) * a.inv_batch;
      g_f2_row_terms[2 * row + 1] = ((__ffs(hit) - 1) == label ? 1.f : 0.f) * a.inv_batch;
    }
    if (a.logits_out && lane < NCLS) a.logits_out[(size_t)row * NCLS + lane] = logit;
    if (a.train && lane < DL_LD) a.dl_out[(size_t)row * DL_LD + lane] = dl_mine;
  }
  {
    __shared__ unsigned int s_last;
    if (arrive_last_cta(&g_f2_ticket, gridDim.x, 1, F2_THREADS, &s_last) && warp == 0) {
      float l = 0.f, h = 0.f;
      for (int r = lane; r < (int)gridDim.x; r += 32) {
        l += __ldcg(g_f2_row_terms + 2 * r);
        h += __ldcg(g_f2_row_terms + 2 * r + 1);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        l += __shfl_xor_sync(0xffffffffu, l, o);
        h += __shfl_xor_sync(0xffffffffu, h, o);
      }
      if (lane == 0) {
        a.loss_acc[0] += l;
        a.loss_acc[1] += h;
      }
    }
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
constexpr int FW_J = 8;
constexpr int FW_ROWS = 256;
__global__ void __launch_bounds__(256) fc2_wgrad_kernel(const float* __restrict__ h,            // [B,512]
                                                        const float* __restrict__ dl,           // [B,12]
                                                        const __nv_bfloat16* __restrict__ dh,   // [B,512]
                                                        float* __restrict__ g_w2, float* __restrict__ g_b2,
                                                        float* __restrict__ g_b1, int B) {
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
    if (kind == 0) g_w2[(size_t)(j0 + oj) * NCLS + oc] = acc;
    else if (kind == 1) g_b1[j0 + oj] = acc;
    else if (kind == 2 && blockIdx.x == 0) g_b2[oc] = acc;
  }
}

// =====================================================================================================
// unpool2: d(pool2 out) [B,7,7,64] (bf16) -> d(conv2 pre-activation) [B,14,14,64] (bf16, dense with zeros),
// plus the conv2 bias gradient.
// =====================================================================================================
__global__ void __launch_bounds__(256) unpool2_kernel(const __nv_bfloat16* __restrict__ dpool,  // [B,3136]
                                                      const uint8_t* __restrict__ code,         // [B,3136]
                                                      __nv_bfloat16* __restrict__ dy,           // [B,14,14,64]
                                                      float* __restrict__ g_bias,               // [64]
                                                      int B) {
  __shared__ float s_gb[64];
  if (threadIdx.x < 64) s_gb[threadIdx.x] = 0.f;
  __syncthreads();
  pdl_wait();
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)
  const int total = B * 49 * 8;   // (b, pooled position, group of 8 channels)
  float gsum[8];                  // bias-gradient partials: a thread keeps the same channel group across trips
#pragma unroll
  for (int j = 0; j < 8; ++j) gsum[j] = 0.f;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    const int cg = t & 7, pos = (t >> 3) % 49, b = (t >> 3) / 49;
    const int ph = pos / 7, pw = pos - ph * 7;
    const size_t src = ((size_t)b * 49 + pos) * 64 + cg * 8;
    const uint4 gv = *reinterpret_cast<const uint4*>(dpool + src);
    const uint2 cv = *reinterpret_cast<const uint2*>(code + src);
    const uint32_t g32[4] = {gv.x, gv.y, gv.z, gv.w};
    uint32_t o[4][4];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int k = 0; k < 4; ++k) o[p][k] = 0u;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t c = ((j < 4 ? cv.x : cv.y) >> ((j & 3) * 8)) & 0xffu;
      const uint32_t half = (g32[j >> 1] >> ((j & 1) * 16)) & 0xffffu;
      if (c & 4u) {
        o[c & 3u][j >> 1] |= half << ((j & 1) * 16);
        gsum[j] += __bfloat162float(__ushort_as_bfloat16((unsigned short)half));
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int y = 2 * ph + (p >> 1), x = 2 * pw + (p & 1);
      *reinterpret_cast<uint4*>(dy + (((size_t)b * 14 + y) * 14 + x) * 64 + cg * 8) =
          make_uint4(o[p][0], o[p][1], o[p][2], o[p][3]);
    }
  }
  // lanes l, l+8, l+16, l+24 of a warp share the channel group: fold them with two shuffles
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    gsum[j] += __shfl_xor_sync(0xffffffffu, gsum[j], 8);
    gsum[j] += __shfl_xor_sync(0xffffffffu, gsum[j], 16);
  }
  if ((threadIdx.x & 31) < 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) atomicAdd(&s_gb[(threadIdx.x & 7) * 8 + j], gsum[j]);
  }
  __syncthreads();
  if (threadIdx.x < 64) atomicAdd(g_bias + threadIdx.x, s_gb[threadIdx.x]);
}

// =====================================================================================================
// conv1 wgrad fused with the backward of maxpool1 + ReLU1.  One CTA per image, lane = channel.
//   dW[tap][c] += img[y+kh-2][x+kw-2] * g   where (y,x) is the argmax position of pooled element g.
// =====================================================================================================
__global__ void __launch_bounds__(256) conv1_wgrad_kernel(const float* __restrict__ images,        // [B,28,28]
                                                          const __nv_bfloat16* __restrict__ dpool, // [B,14,14,32]
                                                          const uint8_t* __restrict__ code,        // [B,14,14,32]
                                                          float* __restrict__ g_w,                 // [25][32]
                                                          float* __restrict__ g_b,                 // [32]
                                                          int B) {
  // Everything an image needs is staged in shared memory with wide coalesced loads first (the loop below
  // would otherwise expose one global-load latency per pooled position).
  __shared__ float s_img[32][34];     // row stride 34: the four argmax positions of a window hit distinct banks
  __shared__ __align__(16) float s_g[8 * 26 * 32];     // [196][32] masked gradients; reused as [8][26][32] for the reduction
  __shared__ __align__(8) uint8_t s_pos[196 * 32];     // argmax position code (bits 0-1)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  pdl_wait();
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)
  float acc[26];
#pragma unroll
  for (int t = 0; t < 26; ++t) acc[t] = 0.f;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * 32; i += blockDim.x) {
      const int r = i >> 5, c = i & 31, y = r - 2, x = c - 2;
      s_img[r][c] = (y >= 0 && y < 28 && x >= 0 && x < 28) ? images[(size_t)b * 784 + y * 28 + x] : 0.f;
    }
    for (int i = threadIdx.x; i < 196 * 4; i += blockDim.x) {   // 8 channels per item
      const size_t o = (size_t)b * 6272 + (size_t)i * 8;
      const uint4 gv = *reinterpret_cast<const uint4*>(dpool + o);
      const uint2 cv = *reinterpret_cast<const uint2*>(code + o);
      const uint32_t g32[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const uint32_t c = ((j < 4 ? cv.x : cv.y) >> ((j & 3) * 8)) & 0xffu;
        const float g = __bfloat162float(__ushort_as_bfloat16((unsigned short)((g32[j >> 1] >> ((j & 1) * 16)) & 0xffffu)));
        s_g[i * 8 + j] = (c & 4u) ? g : 0.f;
      }
      *reinterpret_cast<uint2*>(s_pos + i * 8) = cv;
    }
    __syncthreads();
    for (int pos = warp; pos < 196; pos += 8) {
      const float g = s_g[pos * 32 + lane];
      const uint32_t c = s_pos[pos * 32 + lane];
      const int ph = pos / 14, pw = pos - ph * 14;
      const int y = 2 * ph + ((c >> 1) & 1), x = 2 * pw + (c & 1);   // conv-output coordinates of the max
#pragma unroll
      for (int kh = 0; kh < 5; ++kh)
#pragma unroll
        for (int kw = 0; kw < 5; ++kw) acc[kh * 5 + kw] = fmaf(s_img[y + kh][x + kw], g, acc[kh * 5 + kw]);
      acc[25] += g;
    }
  }
  __syncthreads();
#pragma unroll
  for (int t = 0; t < 26; ++t) s_g[(warp * 26 + t) * 32 + lane] = acc[t];
  __syncthreads();
  for (int i = threadIdx.x; i < 26 * 32; i += blockDim.x) {
    const int t = i >> 5, c = i & 31;
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += s_g[(w * 26 + t) * 32 + c];
    if (t < 25) atomicAdd(g_w + t * 32 + c, s);
    else atomicAdd(g_b + c, s);
  }
}

// bias + ReLU on an fp32 accumulator -> bf16 activations (MLP hidden layers), optionally zeroing the
// accumulator for the next split-K pass.  Backward companion: mask the incoming gradient.
__global__ void bias_relu_bf16_kernel(float* __restrict__ acc, const float* __restrict__ bias,
                                      __nv_bfloat16* __restrict__ out, int rows, int cols, int zero_acc) {
  pdl_wait();
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)
  const long long n = (long long)rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = acc[i] + bias[i % cols];
    if (zero_acc) acc[i] = 0.f;
    out[i] = __float2bfloat16(v > 0.f ? v : 0.f);
  }
}

}  // namespace dm

extern "C" {

// zero0/1/2 (+ counts, in floats): optional regions cleared by the kernel.
int dm_conv1_fwd(const void* images, const void* w, const void* bias, void* out, void* code, int B, void* zero0,
                 int n0, void* zero1, int n1, void* zero2, int n2, void* stream) {
  dm::ZeroRanges zr;
  zr.ptr[0] = reinterpret_cast<float*>(zero0); zr.n[0] = n0;
  zr.ptr[1] = reinterpret_cast<float*>(zero1); zr.n[1] = n1;
  zr.ptr[2] = reinterpret_cast<float*>(zero2); zr.n[2] = n2;
  static const int version = dm::env_int("DMNIST_CONV1_FWD", 2);     // 1: first-generation kernel (kept for A/B runs)
  if (version == 1)
    return (int)dm::launch_kernel(dm::conv1_fwd_kernel, dim3(7 * B), dim3(dm::C1_THREADS), 0, reinterpret_cast<cudaStream_t>(stream),
        reinterpret_cast<const float*>(images), reinterpret_cast<const float*>(w), reinterpret_cast<const float*>(bias),
        reinterpret_cast<__nv_bfloat16*>(out), reinterpret_cast<uint8_t*>(code), zr);
  return (int)dm::launch_kernel(dm::conv1_fwd2_kernel, dim3(7 * B), dim3(dm::C1B_THREADS), 0, reinterpret_cast<cudaStream_t>(stream),
      reinterpret_cast<const float*>(images), reinterpret_cast<const float*>(w), reinterpret_cast<const float*>(bias),
      reinterpret_cast<__nv_bfloat16*>(out), reinterpret_cast<uint8_t*>(code), zr);
}

// Critical-path half: logits / loss / accuracy and (train) dh, h_out, dl_out.  scratch_h [B,512] fp32 and
// scratch_dl [B,12] fp32 are only touched when train != 0.
int dm_fc2_fwd_bwd(const void* h_part, long long part_stride, int splits, const void* b1, const void* w2, const void* b2,
                   const void* labels, void* dh, void* scratch_h, void* scratch_dl, void* loss_acc, void* logits_out,
                   int B, int train, unsigned int seed_mix, const void* step_ptr, float keep_prob, void* stream) {
  if (splits < 1 || splits > dm::F2_MAX_SPLITS || B < 1 || B > dm::F2_MAX_ROWS) return -1;
  dm::Fc2Args a;
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
  a.logits_out = reinterpret_cast<float*>(logits_out);
  a.B = B; a.train = train; a.seed_mix = seed_mix;
  a.step_ptr = reinterpret_cast<const uint32_t*>(step_ptr);
  a.keep_prob = keep_prob;
  a.inv_batch = 1.f / (float)B;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(dm::fc2_fwd_bwd_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  return (int)dm::launch_kernel(dm::fc2_fwd_bwd_kernel, dim3(B), dim3(dm::F2_THREADS), 0,
                                reinterpret_cast<cudaStream_t>(stream), a);
}

// Side-branch half: g_w2 [512][10], g_b2 [10], g_b1 [512] (plain stores).
int dm_fc2_wgrad(const void* scratch_h, const void* scratch_dl, const void* dh, void* g_w2, void* g_b2, void* g_b1, int B,
                 void* stream) {
  // side-branch kernel: it has to share SMs with the tensor-core kernels (max-shared L1 split), see dm_fused_sync_bucket
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(dm::fc2_wgrad_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  return (int)dm::launch_kernel(dm::fc2_wgrad_kernel, dim3(dm::HID / dm::FW_J), dim3(256), 0,
                                reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const float*>(scratch_h),
                                reinterpret_cast<const float*>(scratch_dl), reinterpret_cast<const __nv_bfloat16*>(dh),
                                reinterpret_cast<float*>(g_w2), reinterpret_cast<float*>(g_b2),
                                reinterpret_cast<float*>(g_b1), B);
}

int dm_unpool2(const void* dpool, const void* code, void* dy, void* g_bias, int B, void* stream) {
  int grid = (B * 49 * 8 + 255) / 256;
  if (grid > dm::num_sms() * 2) grid = dm::num_sms() * 2;
  return (int)dm::launch_kernel(dm::unpool2_kernel, dim3(grid), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
      reinterpret_cast<const __nv_bfloat16*>(dpool), reinterpret_cast<const uint8_t*>(code),
      reinterpret_cast<__nv_bfloat16*>(dy), reinterpret_cast<float*>(g_bias), B);
}

int dm_conv1_wgrad(const void* images, const void* dpool, const void* code, void* g_w, void* g_b, int B, void* stream) {
  // one image per CTA (37 KB smem, 57 regs: up to four CTAs share an SM): all B CTAs are resident at once, so the
  // staging latency of one overlaps the accumulation loop of its neighbours instead of serialising per image
  int grid = B < dm::num_sms() * 4 ? B : dm::num_sms() * 4;
  return (int)dm::launch_kernel(dm::conv1_wgrad_kernel, dim3(grid), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
      reinterpret_cast<const float*>(images), reinterpret_cast<const __nv_bfloat16*>(dpool),
      reinterpret_cast<const uint8_t*>(code), reinterpret_cast<float*>(g_w), reinterpret_cast<float*>(g_b), B);
}

int dm_bias_relu_bf16(void* acc, const void* bias, void* out, int rows, int cols, int zero_acc, void* stream) {
  long long n = (long long)rows * cols;
  int grid = (int)((n + 255) / 256 < dm::num_sms() * 8 ? (n + 255) / 256 : dm::num_sms() * 8);
  dm::bias_relu_bf16_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<float*>(acc), reinterpret_cast<const float*>(bias), reinterpret_cast<__nv_bfloat16*>(out), rows,
      cols, zero_acc);
  return (int)cudaGetLastError();
}

}  // extern "C"
