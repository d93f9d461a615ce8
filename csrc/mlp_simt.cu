// SIMT kernels of the MLP models (BASELINE.json configs: 2-layer plumbing MLP, 3-layer MLP at batch
// 8192/replica).  Hidden layers run on the wgmma GEMM (csrc/gemm_tc.cu, bias+ReLU fused in its
// epilogue); what is left for CUDA cores:
//   dense10_xent     last layer (H -> 10, too narrow for a TMA/UMMA operand: 20-byte rows) + softmax-CE +
//                    accuracy, and backward to d(hidden) with the ReLU mask applied; the output-layer
//                    weights stay resident in shared memory for all rows of the CTA
//   relu_bwd_colsum  dpre = dh * (h > 0) (bf16) and the bias gradient (column sums) in one pass
//   f32 -> bf16      input conversion (dm_f32_to_bf16 in fused_sync.cu)
#include "common.cuh"
#include "host_utils.h"

namespace dm {

constexpr int XN = 10;            // classes
constexpr int XN_PAD = 64;        // dl is also written as a zero-padded [B,64] bf16 matrix: the B operand
                                  // of the wgmma GEMM that forms the output-layer weight gradient
constexpr int X_WARPS = 8;

struct XentArgs {
  const __nv_bfloat16* h;     // [B,H] last hidden activations (post ReLU)
  const float* w;             // [H,10]
  const float* b;             // [10]
  const long long* labels;    // [B]
  __nv_bfloat16* dh;          // [B,H]  d loss / d (pre-activation of the last hidden layer)   (train)
  __nv_bfloat16* dl_pad;      // [B,64] dlogits, columns 10..63 stay zero                       (train)
  float* g_b;                 // [10] (pre-zeroed)
  float* loss_acc;            // [2]  (pre-zeroed)
  float* logits_out;          // optional [B,10]
  int B, H, train;
  float inv_batch;
};

__global__ void __launch_bounds__(X_WARPS * 32) dense10_xent_kernel(XentArgs a) {
  extern __shared__ float s_w[];                  // [H][11]: pitch 11 keeps lane-strided reads conflict-free
  __shared__ float s_gb[XN];
  for (int i = threadIdx.x; i < a.H * XN; i += blockDim.x) s_w[(i / XN) * 11 + (i % XN)] = a.w[i];
  if (threadIdx.x < XN) s_gb[threadIdx.x] = 0.f;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float gb_local[XN];
#pragma unroll
  for (int c = 0; c < XN; ++c) gb_local[c] = 0.f;
  for (int row = blockIdx.x * X_WARPS + warp; row < a.B; row += gridDim.x * X_WARPS) {
    const __nv_bfloat16* hr = a.h + (size_t)row * a.H;
    float acc[XN];
#pragma unroll
    for (int c = 0; c < XN; ++c) acc[c] = 0.f;
#pragma unroll 4
    for (int j = lane; j < a.H; j += 32) {
      const float hv = __bfloat162float(hr[j]);
#pragma unroll
      for (int c = 0; c < XN; ++c) acc[c] = fmaf(hv, s_w[j * 11 + c], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < XN; ++c) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
      acc[c] += a.b[c];
    }
    const int label = (int)a.labels[row];
    float m = acc[0];
    int arg = 0;
#pragma unroll
    for (int c = 1; c < XN; ++c)
      if (acc[c] > m) { m = acc[c]; arg = c; }
    float p[XN], s = 0.f, l_label = 0.f;
#pragma unroll
    for (int c = 0; c < XN; ++c) { p[c] = __expf(acc[c] - m); s += p[c]; if (c == label) l_label = acc[c]; }
    const float inv_s = 1.f / s;
    if (lane == 0) {
      atomicAdd(a.loss_acc + 0, (__logf(s) - (l_label - m)) * a.inv_batch);
      atomicAdd(a.loss_acc + 1, (arg == label ? 1.f : 0.f) * a.inv_batch);
    }
    if (a.logits_out && lane < XN) {
      float v = 0.f;
#pragma unroll
      for (int c = 0; c < XN; ++c) if (c == lane) v = acc[c];
      a.logits_out[(size_t)row * XN + lane] = v;
    }
    if (!a.train) continue;
    float dl[XN];
#pragma unroll
    for (int c = 0; c < XN; ++c) {
      dl[c] = (p[c] * inv_s - (c == label ? 1.f : 0.f)) * a.inv_batch;
      gb_local[c] += dl[c];                      // identical on every lane; lane 0 publishes below
    }
    if (lane < 16) {
      float v = 0.f;
#pragma unroll
      for (int c = 0; c < XN; ++c) if (c == lane) v = dl[c];
      a.dl_pad[(size_t)row * XN_PAD + lane] = __float2bfloat16(v);
    }
    __nv_bfloat16* dr = a.dh + (size_t)row * a.H;
#pragma unroll 4
    for (int j = lane; j < a.H; j += 32) {
      float d = 0.f;
#pragma unroll
      for (int c = 0; c < XN; ++c) d = fmaf(dl[c], s_w[j * 11 + c], d);
      dr[j] = __float2bfloat16(__bfloat162float(hr[j]) > 0.f ? d : 0.f);   // ReLU mask of the producing layer
    }
  }
  if (!a.train) return;
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < XN; ++c) atomicAdd(&s_gb[c], gb_local[c]);
  }
  __syncthreads();
  if (threadIdx.x < XN) atomicAdd(a.g_b + threadIdx.x, s_gb[threadIdx.x]);
}

// dpre[b][j] = dh[b][j] * (h[b][j] > 0) (in place when dpre == dh; h may be null = no mask), and
// g_bias[j] += sum_b dpre[b][j].  CTA = 64 columns x a slab of rows; 256 threads = 32 column pairs x 8 row lanes.
__global__ void __launch_bounds__(256) relu_bwd_colsum_kernel(const __nv_bfloat16* __restrict__ dh,
                                                              const __nv_bfloat16* __restrict__ h,
                                                              __nv_bfloat16* __restrict__ dpre,
                                                              float* __restrict__ g_bias, int B, int H, int rows_per_cta) {
  __shared__ float s_sum[8][64];
  const int cp = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col = blockIdx.x * 64 + cp * 2;
  const int r0 = blockIdx.y * rows_per_cta, r1 = min(r0 + rows_per_cta, B);
  float s0 = 0.f, s1 = 0.f;
  if (col < H) {
    for (int r = r0 + rl; r < r1; r += 8) {
      const size_t o = (size_t)r * H + col;
      const __nv_bfloat162 d = *reinterpret_cast<const __nv_bfloat162*>(dh + o);
      float d0 = __low2float(d), d1 = __high2float(d);
      if (h != nullptr) {
        const __nv_bfloat162 hv = *reinterpret_cast<const __nv_bfloat162*>(h + o);
        d0 = __low2float(hv) > 0.f ? d0 : 0.f;
        d1 = __high2float(hv) > 0.f ? d1 : 0.f;
        *reinterpret_cast<uint32_t*>(dpre + o) = pack_bf16x2(d0, d1);
      }
      s0 += d0;
      s1 += d1;
    }
  }
  s_sum[rl][cp * 2] = s0;
  s_sum[rl][cp * 2 + 1] = s1;
  __syncthreads();
  if (threadIdx.x < 64 && blockIdx.x * 64 + threadIdx.x < H) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += s_sum[i][threadIdx.x];
    atomicAdd(g_bias + blockIdx.x * 64 + threadIdx.x, s);
  }
}

}  // namespace dm

extern "C" {

int dm_dense10_xent(const void* h, const void* w, const void* b, const void* labels, void* dh, void* dl_pad, void* g_b,
                    void* loss_acc, void* logits_out, int B, int H, int train, void* stream) {
  using namespace dm;
  XentArgs a;
  a.h = reinterpret_cast<const __nv_bfloat16*>(h);
  a.w = reinterpret_cast<const float*>(w);
  a.b = reinterpret_cast<const float*>(b);
  a.labels = reinterpret_cast<const long long*>(labels);
  a.dh = reinterpret_cast<__nv_bfloat16*>(dh);
  a.dl_pad = reinterpret_cast<__nv_bfloat16*>(dl_pad);
  a.g_b = reinterpret_cast<float*>(g_b);
  a.loss_acc = reinterpret_cast<float*>(loss_acc);
  a.logits_out = reinterpret_cast<float*>(logits_out);
  a.B = B; a.H = H; a.train = train;
  a.inv_batch = 1.f / (float)B;
  const int smem = H * 11 * 4;
  if (smem > 220 * 1024) return -2;
  DM_CUDA_OK(cudaFuncSetAttribute(dense10_xent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int grid = (B + X_WARPS - 1) / X_WARPS;
  if (grid > dm::num_sms()) grid = dm::num_sms();
  dense10_xent_kernel<<<grid, X_WARPS * 32, smem, reinterpret_cast<cudaStream_t>(stream)>>>(a);
  return (int)cudaGetLastError();
}

int dm_relu_bwd_colsum(const void* dh, const void* h, void* dpre, void* g_bias, int B, int H, void* stream) {
  if (H & 1) return -1;
  int slabs = (B + 255) / 256;
  if (slabs > 64) slabs = 64;
  const int rows = (B + slabs - 1) / slabs;
  dim3 grid((H + 63) / 64, slabs);
  dm::relu_bwd_colsum_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(dh), reinterpret_cast<const __nv_bfloat16*>(h),
      reinterpret_cast<__nv_bfloat16*>(dpre), reinterpret_cast<float*>(g_bias), B, H, rows);
  return (int)cudaGetLastError();
}

}  // extern "C"
