// wgmma GEMM for sm_90a:  D[M,N] (+)= A[M,K] * B[K,N],  bf16 in, fp32 accumulate in registers.
//
// Covers every dense GEMM of the models (reference ops K6/K8: tf.matmul, src/mnist.py:136,145,
// and their gradients) without a single transpose kernel: each operand may be K-major or
// MN-major in memory, so the TF layouts ([in,out] weights, [batch,features] activations) are
// consumed as they are:
//     fc fwd    D[b,out]  = X[b,in]   (A K-major)  * W[in,out]  (B MN-major)
//     fc dgrad  D[b,in]   = dY[b,out] (A K-major)  * W[in,out]  (B K-major:  rows=in, K=out contiguous)
//     fc wgrad  D[in,out] = X[b,in]   (A MN-major) * dY[b,out]  (B MN-major),  K = batch
//
// Structure (one 128 x BN output tile per CTA, optional split-K over gridDim.z):
//     warps 0-7   two consumer warpgroups: warpgroup g issues wgmma for rows 64 g .. 64 g + 63 of the tile
//                 (BN / 64 m64n64k16 instructions per K step); afterwards all eight warps run the epilogue
//     warp 8      TMA producer      cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx
// The accumulator is staged through the (then idle) operand ring as a [128][BN] fp32 tile, so the epilogue
// keeps one thread per output row with 32 consecutive columns in registers.
#include "common.cuh"
#include "host_utils.h"

namespace dm {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_STAGES = 4;
constexpr int GEMM_CONSUMERS = 256;                   // two warpgroups
constexpr int GEMM_THREADS = GEMM_CONSUMERS + 32;      // + the TMA producer warp

enum GemmEpilogue : int { EPI_STORE_F32 = 0, EPI_ATOMIC_F32 = 1, EPI_STORE_BF16 = 2, EPI_BIAS_RELU_BF16 = 3,
                          // fc1 dgrad fused with the backward of maxpool2 + ReLU2 (reference K4/K3 gradients): a 64-column
                          // tile is one pooled position x 64 channels; the epilogue scatters each value to the argmax
                          // pixel of its 2x2 window (dense bf16 [B,14,14,64], zeros elsewhere) and reduces the conv2
                          // bias gradient -- the separate unpool kernel and the [B,3136] intermediate disappear.
                          EPI_UNPOOL2_BF16 = 4,
                          // fc weight gradient with L2 decay (--weight_decay): each element is fma(decay, W, acc) with one
                          // rounding (then rounded to bf16 for the wire variant), W the fp32 weights in the output's layout;
                          // each CTA also stores the sum of its tile's W^2, in double and a fixed order, into decay_part
                          EPI_STORE_F32_DECAY = 5, EPI_STORE_BF16_DECAY = 6 };

struct GemmParams {
  int M, N;        // logical output extent (predication)
  int num_kb;      // ceil(K / 64)
  int ldo;         // output leading dimension (elements)
  void* out;
  long long split_stride;   // EPI_STORE_F32 with split-K: split z writes its partial tile at out + z*split_stride
  const float* bias;        // EPI_BIAS_RELU_BF16: per-column bias (reference K2/K3 fused into the producer)
  const uint8_t* code;      // EPI_UNPOOL2_BF16: pooling codes [M][N] (bits 0-1 argmax position, bit 2 ReLU active)
  float* bias_part;         // EPI_UNPOOL2_BF16: [CTAs][64] conv2 bias-gradient partials, one slot per CTA
  const float* decay_w;     // EPI_*_DECAY: fp32 weights [M][ldo]
  double* decay_part;       // EPI_*_DECAY: one W^2 partial per CTA, at blockIdx.y * gridDim.x + blockIdx.x
  float decay;              // EPI_*_DECAY: lambda
};

template <int BN>
struct GemmSmem {
  static constexpr int A_BYTES = GEMM_BM * GEMM_BK * 2;   // 16 KB
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = GEMM_STAGES;
  static constexpr int BAR_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BPART_OFFSET = BAR_OFFSET + 128;   // EPI_UNPOOL2_BF16: [4 row quarters][64] bias partials
  static constexpr int TOTAL = BAR_OFFSET + 2048 + 1024;  // barriers, bias partials + alignment slack
  // epilogue staging (reuses the ring): rows padded by 4 floats so that 32 threads reading 16 B of 32 different rows
  // hit distinct banks
  static constexpr int ACC_LD = BN + 4;
  static_assert(GEMM_BM * ACC_LD * 4 <= BAR_OFFSET, "accumulator staging must fit in the operand ring");
};

// EPI_UNPOOL2_BF16: each CTA stores its conv2 bias-gradient partials to its own slot, and a later kernel adds the slots up
// in CTA order (add_ordered_slot_sum64), so the result does not depend on the order in which the CTAs finish, and nothing
// waits for the sum before the data gradient is out.
constexpr int UNPOOL_MAX_CTAS = 4096;                  // batch <= 4096 / 49 row tiles x 128 = 10 624 rows
// The slots of dm_fc1_dgrad_unpool, which sums them right after the GEMM: one launch pair in flight per device.
__device__ float g_unpool_bias_part[UNPOOL_MAX_CTAS * 64];

int fc1_dgrad_unpool_max_batch() { return UNPOOL_MAX_CTAS / (3136 / 64) * GEMM_BM; }

int unpool_bias_slots(int B) { return (B + GEMM_BM - 1) / GEMM_BM * (3136 / 64); }

// g_bias += the slots' sum in slot order: 16 CTAs, CTA q adds channels 4q .. 4q + 3
__global__ void __launch_bounds__(64) unpool_bias_sum_kernel(const float* slots, int n, float* g_bias) {
  __shared__ float4 s_buf[4 * 64];
  pdl_wait();
  add_ordered_slot_sum64<64>(slots, n, blockIdx.x, g_bias, s_buf);
}

template <int BN, bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmParams p) {
  using S = GemmSmem<BN>;
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle atoms repeat every 1024 B: align the ring so descriptors need no base offset.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::BAR_OFFSET);
  uint64_t* empty_bar = full_bar + S::STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * GEMM_BM;
  const int n0 = blockIdx.y * BN;
  // split-K: this CTA owns k-blocks [kb_begin, kb_end)
  const int kb_begin = (int)(((long long)p.num_kb * blockIdx.z) / gridDim.z);
  const int kb_end = (int)(((long long)p.num_kb * (blockIdx.z + 1)) / gridDim.z);
  const int nkb = kb_end - kb_begin;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < S::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], GEMM_CONSUMERS / 32);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();      // everything above is private set-up; operands / outputs belong to earlier kernels until here
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)

  if (warp == 8) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % S::STAGES;
        const uint32_t ph = (i / S::STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* sA = smem + s * S::STAGE_BYTES;
        uint8_t* sB = sA + S::A_BYTES;
        mbar_expect_tx(&full_bar[s], S::STAGE_BYTES);
        const int k0 = (kb_begin + i) * GEMM_BK;
        if (!A_MN) {
          tma_load_2d(sA, &tmA, &full_bar[s], k0, m0);                 // box {64 k, 128 m}
        } else {
          tma_load_2d(sA, &tmA, &full_bar[s], m0, k0);                 // box {64 m, 64 k}
          tma_load_2d(sA + 8192, &tmA, &full_bar[s], m0 + 64, k0);
        }
        if (!B_MN) {
          tma_load_2d(sB, &tmB, &full_bar[s], k0, n0);                 // box {64 k, BN n}
        } else {
#pragma unroll
          for (int j = 0; j < BN / 64; ++j) tma_load_2d(sB + j * 8192, &tmB, &full_bar[s], n0 + 64 * j, k0);
        }
      }
    }
    return;
  }

  // ------------------------------ consumers: wgmma main loop ------------------------------
  const int wg = warp >> 2;                        // warpgroup = rows 64 wg .. 64 wg + 63 of the tile
  constexpr int NC = BN / 64;                      // 64-column chunks
  float acc[NC][32];
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[c][j] = 0.f;
  for (int i = 0; i < nkb; ++i) {
    const int s = i % S::STAGES;
    mbar_wait(&full_bar[s], (i / S::STAGES) & 1);
    const uint32_t a_addr = smem_u32(smem + s * S::STAGE_BYTES);
    const uint32_t b_addr = a_addr + S::A_BYTES;
    // K-major:  128 B rows (64 bf16 of K), 8-row groups 1024 B apart; K advances 32 B per K step of 16.
    // MN-major: 128 B k-rows (64 bf16 of M/N), 8-k groups 1024 B apart, 64-wide M/N chunks 8192 B
    //           apart; K advances 16 k-rows = 2048 B per K step.
    // Either way rows 64 .. 127 of A and columns 64 c .. 64 c + 63 of B start 8192 B further on.
    const uint64_t da0 = A_MN ? make_smem_desc(a_addr + 8192 * wg, 8192, 1024, SWZ_128B)
                              : make_smem_desc(a_addr + 8192 * wg, 16, 1024, SWZ_128B);
    const uint64_t db0 = B_MN ? make_smem_desc(b_addr, 8192, 1024, SWZ_128B)
                              : make_smem_desc(b_addr, 16, 1024, SWZ_128B);
#pragma unroll
    for (int c = 0; c < NC; ++c) fence_regs(acc[c]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GEMM_BK / 16; ++k) {
      const uint64_t da = desc_advance(da0, (A_MN ? 2048u : 32u) * k);
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const uint64_t db = desc_advance(db0, (B_MN ? 2048u : 32u) * k + 8192u * c);
        wgmma_m64n64_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[c], da, db, (i | k) != 0);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NC; ++c) fence_regs(acc[c]);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);     // stage reusable: this warp's MMAs have read it
  }

  // ------------------------------ accumulator -> shared staging tile ------------------------------
  named_bar_sync(1, GEMM_CONSUMERS);               // both warpgroups are done with the ring
  float* stage = reinterpret_cast<float*>(smem);
  {
    const int r = 16 * warp + (lane >> 2);         // tile row of d[4j], d[4j+1]; d[4j+2], d[4j+3] are 8 rows below
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = 64 * c + 8 * j + 2 * (lane & 3);
        *reinterpret_cast<float2*>(stage + r * S::ACC_LD + col) = make_float2(acc[c][4 * j], acc[c][4 * j + 1]);
        *reinterpret_cast<float2*>(stage + (r + 8) * S::ACC_LD + col) = make_float2(acc[c][4 * j + 2], acc[c][4 * j + 3]);
      }
  }
  named_bar_sync(1, GEMM_CONSUMERS);

  if (EPI == EPI_STORE_F32 && n0 + BN <= p.N && (p.ldo & 3) == 0) {
    // plain fp32 store of a full-width tile (the fc1 forward's split partials): whole rows from the staging tile, BN / 4
    // consecutive lanes per row, so a warp instruction writes whole 128-byte lines instead of 16 bytes into each of 32
    float* o = reinterpret_cast<float*>(p.out) + (size_t)blockIdx.z * p.split_stride + n0;
    constexpr int F4_PER_ROW = BN / 4;
#pragma unroll 4
    for (int i = threadIdx.x; i < GEMM_BM * F4_PER_ROW; i += GEMM_CONSUMERS) {
      const int lr = i / F4_PER_ROW, j = i % F4_PER_ROW;
      if (m0 + lr < p.M)
        *reinterpret_cast<float4*>(o + (size_t)(m0 + lr) * p.ldo + 4 * j) = *reinterpret_cast<const float4*>(stage + lr * S::ACC_LD + 4 * j);
    }
    return;
  }

  // ------------------------------ epilogue: thread = tile row, 32-column chunks ------------------------------
  constexpr bool DECAY = EPI == EPI_STORE_F32_DECAY || EPI == EPI_STORE_BF16_DECAY;
  double wsq = 0.0;                                  // DECAY: sum of this thread's W^2, chunk by chunk, column by column
  {
    const int lr = threadIdx.x & 127;                // tile row
    const int half = threadIdx.x >> 7;               // chunks half, half + 2, ...
    const int row = m0 + lr;
    const int c_begin = half;
    const int c_end = EPI == EPI_UNPOOL2_BF16 ? c_begin + 1 : BN / 32;
    uint32_t cw[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
    if (EPI == EPI_UNPOOL2_BF16 && row < p.M) {
      // pooling codes of this thread's 32 channels
      const uint4* cp = reinterpret_cast<const uint4*>(p.code + (size_t)row * p.N + n0 + c_begin * 32);
      const uint4 c0 = __ldg(cp), c1 = __ldg(cp + 1);
      cw[0] = c0.x; cw[1] = c0.y; cw[2] = c0.z; cw[3] = c0.w; cw[4] = c1.x; cw[5] = c1.y; cw[6] = c1.z; cw[7] = c1.w;
    }
#pragma unroll 1
    for (int c = c_begin; c < c_end; c += 2) {
      uint32_t v[32];
      {
        const float* src = stage + lr * S::ACC_LD + c * 32;
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float4 t = *reinterpret_cast<const float4*>(src + j);
          v[j] = __float_as_uint(t.x); v[j + 1] = __float_as_uint(t.y);
          v[j + 2] = __float_as_uint(t.z); v[j + 3] = __float_as_uint(t.w);
        }
      }
      const int col0 = n0 + c * 32;
      if (DECAY && row < p.M) {
        // the W tile is read once: for the lambda * W term and for the W^2 partial
        const float* wp = p.decay_w + (size_t)row * p.ldo + col0;
        float w[32];
        if (col0 + 32 <= p.N && (p.ldo & 3) == 0) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(wp + j));
            w[j] = t.x; w[j + 1] = t.y; w[j + 2] = t.z; w[j + 3] = t.w;
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) w[j] = col0 + j < p.N ? __ldg(wp + j) : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          v[j] = __float_as_uint(fma_rn(p.decay, w[j], __uint_as_float(v[j])));
          wsq += (double)w[j] * (double)w[j];        // the product of two floats is exact in double
        }
      }
      if (row < p.M) {
        if (EPI == EPI_STORE_F32 || EPI == EPI_STORE_F32_DECAY) {
          float* o = reinterpret_cast<float*>(p.out) + (size_t)blockIdx.z * p.split_stride + (size_t)row * p.ldo + col0;
          if (col0 + 32 <= p.N && (p.ldo & 3) == 0) {
#pragma unroll
            for (int j = 0; j < 32; j += 4)
              *reinterpret_cast<float4*>(o + j) = make_float4(__uint_as_float(v[j]), __uint_as_float(v[j + 1]),
                                                               __uint_as_float(v[j + 2]), __uint_as_float(v[j + 3]));
          } else {
            for (int j = 0; j < 32; ++j)
              if (col0 + j < p.N) o[j] = __uint_as_float(v[j]);
          }
        } else if (EPI == EPI_ATOMIC_F32) {
          float* o = reinterpret_cast<float*>(p.out) + (size_t)row * p.ldo + col0;
          if (col0 + 32 <= p.N && (p.ldo & 3) == 0) {
#pragma unroll
            for (int j = 0; j < 32; j += 4)
              red_add_f32x4(o + j, __uint_as_float(v[j]), __uint_as_float(v[j + 1]), __uint_as_float(v[j + 2]),
                            __uint_as_float(v[j + 3]));
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (col0 + j < p.N) atomicAdd(o + j, __uint_as_float(v[j]));
          }
        } else if (EPI == EPI_UNPOOL2_BF16) {
          // handled below (needs the whole warp, also for rows beyond M)
        } else {
          if (EPI == EPI_BIAS_RELU_BF16) {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const float b = (col0 + j < p.N) ? __ldg(p.bias + col0 + j) : 0.f;
              v[j] = __float_as_uint(fmaxf(__uint_as_float(v[j]) + b, 0.f));
            }
          }
          __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + (size_t)row * p.ldo + col0;
          if (col0 + 32 <= p.N && (p.ldo & 7) == 0) {
#pragma unroll
            for (int j = 0; j < 32; j += 8) {
              uint4 w;
              w.x = pack_bf16x2(__uint_as_float(v[j]), __uint_as_float(v[j + 1]));
              w.y = pack_bf16x2(__uint_as_float(v[j + 2]), __uint_as_float(v[j + 3]));
              w.z = pack_bf16x2(__uint_as_float(v[j + 4]), __uint_as_float(v[j + 5]));
              w.w = pack_bf16x2(__uint_as_float(v[j + 6]), __uint_as_float(v[j + 7]));
              *reinterpret_cast<uint4*>(o + j) = w;
            }
          } else {
            for (int j = 0; j < 32; ++j)
              if (col0 + j < p.N) o[j] = __float2bfloat16(__uint_as_float(v[j]));
          }
        }
      }
      if (EPI == EPI_UNPOOL2_BF16) {
        // thread = batch row, 32 consecutive channels (ch0 ..) of pooled position `pos`
        const int pos = col0 >> 6, ch0 = col0 & 63;
        const int ph = pos / 7, pw = pos - ph * 7;
        float gs[32];                                   // masked gradient (bias-gradient contribution)
        // The tile's 128 rows x 4 pixels x 64 channels are staged in the (idle) ring, 512 B per row, and then stored a
        // row per warp instruction: 4 whole 128-byte lines (a lane per row would write 16 B into each of 32 lines per
        // instruction, and the stores would take most of the kernel's time).
        // 16-byte chunk j = 8 q4 + 4 half + k of row r sits at j ^ (r & 7): staging and reading are conflict-free.
        uint4* s_dy = reinterpret_cast<uint4*>(smem);
        named_bar_sync(1, GEMM_CONSUMERS);              // every thread has read its accumulator row from the ring
        if (row < p.M) {
          // code byte = argmax position (bits 0-1) | ReLU active (bit 2).  Byte-parallel: for window position q4,
          // x = (codes & 7) ^ (4 | q4) is zero exactly in the matching bytes; x + 0x7f sets bit 7 of the others
          // (no carries: x < 8), so ~(x + 0x7f..) & 0x80.. flags the matches and PRMT's sign-replicate mode widens
          // each flag to a 16-bit lane mask for the packed bf16 pairs.
          uint32_t pk[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) pk[j] = pack_bf16x2(__uint_as_float(v[2 * j]), __uint_as_float(v[2 * j + 1]));
#pragma unroll
          for (int j = 0; j < 32; ++j) gs[j] = ((cw[j >> 2] >> ((j & 3) * 8)) & 4u) ? __uint_as_float(v[j]) : 0.f;
#pragma unroll
          for (int q4 = 0; q4 < 4; ++q4) {              // the four pixels of the 2x2 window: 64 B each
            uint32_t o[16];
#pragma unroll
            for (int w8 = 0; w8 < 8; ++w8) {            // code word w8 <-> channels 4*w8 .. 4*w8+3 <-> pk[2*w8], pk[2*w8+1]
              const uint32_t xz = (cw[w8] & 0x07070707u) ^ (0x04040404u | (0x01010101u * (uint32_t)q4));
              const uint32_t hit = ~(xz + 0x7f7f7f7fu) & 0x80808080u;
              o[2 * w8] = pk[2 * w8] & prmt(hit, 0u, 0x9988u);          // bytes {0,0,1,1} sign-replicated
              o[2 * w8 + 1] = pk[2 * w8 + 1] & prmt(hit, 0u, 0xbbaau);  // bytes {2,2,3,3}
            }
#pragma unroll
            for (int k = 0; k < 4; ++k)
              s_dy[lr * 32 + ((8 * q4 + 4 * half + k) ^ (lr & 7))] = make_uint4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]);
          }
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) gs[j] = 0.f;
        }
        named_bar_sync(1, GEMM_CONSUMERS);
        {
          __nv_bfloat16* dy = reinterpret_cast<__nv_bfloat16*>(p.out);
          const int q4 = lane >> 3, cc = lane & 7;      // pixel of the window, 16-byte chunk of its 64 channels
          const int y = 2 * ph + (q4 >> 1), x = 2 * pw + (q4 & 1);
#pragma unroll 4
          for (int r = warp; r < GEMM_BM; r += GEMM_CONSUMERS / 32)
            if (m0 + r < p.M)
              *reinterpret_cast<uint4*>(dy + (((size_t)(m0 + r) * 14 + y) * 14 + x) * 64 + 8 * cc) = s_dy[r * 32 + (lane ^ (r & 7))];
        }
        // column sums over the warp's 32 rows: butterfly transpose-reduce (31 shuffles), lane l ends with channel ch0 + l
#pragma unroll
        for (int st = 0; st < 5; ++st) {
          const int off = 16 >> st;                     // compile-time after unrolling: gs[] stays in registers
          const bool upper = (lane & off) != 0;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            if (i < off) {
              const float send = upper ? gs[i] : gs[i + off];
              const float keep = upper ? gs[i + off] : gs[i];
              gs[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
          }
        }
        reinterpret_cast<float*>(smem + S::BPART_OFFSET)[((threadIdx.x >> 5) & 3) * 64 + ch0 + lane] = gs[0];
      }
    }
  }
  if (EPI == EPI_UNPOOL2_BF16) {
    const float* s_bpart = reinterpret_cast<const float*>(smem + S::BPART_OFFSET);
    named_bar_sync(1, GEMM_CONSUMERS);
    const int cta = blockIdx.y * gridDim.x + blockIdx.x;
    if (threadIdx.x < 64)
      p.bias_part[cta * 64 + threadIdx.x] =
          s_bpart[threadIdx.x] + s_bpart[64 + threadIdx.x] + s_bpart[128 + threadIdx.x] + s_bpart[192 + threadIdx.x];
  }
  if (DECAY) {
    // the CTA's W^2 partial: a fixed butterfly per warp, then the eight warps in order
    double* s_wsq = reinterpret_cast<double*>(smem + S::BPART_OFFSET);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wsq += __shfl_xor_sync(0xffffffffu, wsq, o);
    if (lane == 0) s_wsq[warp] = wsq;
    named_bar_sync(1, GEMM_CONSUMERS);
    if (threadIdx.x == 0) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < GEMM_CONSUMERS / 32; ++w) s += s_wsq[w];
      p.decay_part[blockIdx.y * gridDim.x + blockIdx.x] = s;
    }
  }

}

// ---------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------
template <int BN, bool A_MN, bool B_MN, int EPI>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int splits,
                       cudaStream_t stream) {
  auto kern = gemm_tc_kernel<BN, A_MN, B_MN, EPI>;
  constexpr int smem = GemmSmem<BN>::TOTAL;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  dim3 grid((p.M + GEMM_BM - 1) / GEMM_BM, (p.N + BN - 1) / BN, splits);
  return (int)launch_kernel(kern, grid, dim3(GEMM_THREADS), smem, stream, tmA, tmB, p);
}

template <int BN, int EPI>
static int dispatch_major(bool a_mn, bool b_mn, const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p,
                          int splits, cudaStream_t stream) {
  if (!a_mn && !b_mn) return launch_gemm<BN, false, false, EPI>(tmA, tmB, p, splits, stream);
  if (!a_mn && b_mn) return launch_gemm<BN, false, true, EPI>(tmA, tmB, p, splits, stream);
  if (a_mn && !b_mn) return launch_gemm<BN, true, false, EPI>(tmA, tmB, p, splits, stream);
  return launch_gemm<BN, true, true, EPI>(tmA, tmB, p, splits, stream);
}

}  // namespace dm

// D[M,N] = A * B with bf16 operands.
//   a_mn == 0: A is [M rows][K cols] (lda elements between rows);   a_mn == 1: A is [K rows][M cols].
//   b_mn == 0: B is [N rows][K cols] (ldb);                          b_mn == 1: B is [K rows][N cols].
//   epi: 0 store fp32, 1 atomicAdd fp32 (split-K; caller zeroes), 2 store bf16, 3 bias+ReLU -> bf16.   bn: 64, 128 or 256.
//   split-K without atomics: epi 0 with splits > 1 and split_stride > 0 -> partial sums at out + z*split_stride
//   (the consumer adds the `splits` partials while loading).
extern "C" int dm_gemm_bf16(const void* A, const void* B, void* out, int M, int N, int K, int lda, int ldb, int ldo,
                            int a_mn, int b_mn, int epi, int splits, int bn, long long split_stride, const void* bias,
                            void* stream_) {
  using namespace dm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if ((bn != 64 && bn != 128 && bn != 256) || epi < 0 || epi > 3 || splits < 1) return -1;
  if (epi == EPI_BIAS_RELU_BF16 && bias == nullptr) return -4;
  if (splits > 1 && !(epi == EPI_ATOMIC_F32 || (epi == EPI_STORE_F32 && split_stride > 0))) return -2;
  if ((lda & 7) || (ldb & 7)) return -3;   // TMA: global strides are multiples of 16 bytes
  CUtensorMap tmA, tmB;
  int rc;
  if (!a_mn) rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, 64, 128, 128);
  else       rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, 64, 128);
  if (rc) return 100 + rc;
  if (!b_mn) rc = make_tmap_2d_bf16(&tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 64, (uint32_t)bn, 128);
  else       rc = make_tmap_2d_bf16(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, 64, 128);
  if (rc) return 200 + rc;
  GemmParams p{M, N, (K + GEMM_BK - 1) / GEMM_BK, ldo, out, splits > 1 ? split_stride : 0,
               reinterpret_cast<const float*>(bias), nullptr, nullptr};
  if (splits > p.num_kb && epi == EPI_ATOMIC_F32) splits = p.num_kb > 0 ? p.num_kb : 1;
#define DM_DISPATCH(BN_, EPI_) return dispatch_major<BN_, EPI_>(a_mn != 0, b_mn != 0, tmA, tmB, p, splits, stream)
  if (bn == 64) {
    if (epi == 0) DM_DISPATCH(64, 0);
    if (epi == 1) DM_DISPATCH(64, 1);
    if (epi == 2) DM_DISPATCH(64, 2);
    DM_DISPATCH(64, 3);
  } else if (bn == 128) {
    if (epi == 0) DM_DISPATCH(128, 0);
    if (epi == 1) DM_DISPATCH(128, 1);
    if (epi == 2) DM_DISPATCH(128, 2);
    DM_DISPATCH(128, 3);
  } else {
    // 128 x 256 tiles: twice the FLOPs per operand byte fetched from L2 (the large MLP GEMMs are L2->SM bandwidth bound with
    // 128 x 128 tiles: 2048 CTAs x 2 MB of operands each)
    if (epi == 0) DM_DISPATCH(256, 0);
    if (epi == 2) DM_DISPATCH(256, 2);
    if (epi == 3) DM_DISPATCH(256, 3);
    return -1;
  }
#undef DM_DISPATCH
}

// fc weight gradient with L2 decay:  D[M,N] = A^T B + decay * W,  A [K rows][M cols] and B [K rows][N cols] bf16 (both
// MN-major, K = batch), 128 x 128 tiles, no split-K.  W: fp32 [M][ldo], the layout of the output.  bf16_out: store bf16
// (the bucketed aggregation's wire buffer) instead of fp32.  decay_part receives dm_gemm_decay_ctas(M, N) doubles, the
// W^2 sum of each CTA's tile.
extern "C" int dm_gemm_decay_ctas(int M, int N) {
  return ((M + dm::GEMM_BM - 1) / dm::GEMM_BM) * ((N + 127) / 128);
}

extern "C" int dm_gemm_bf16_decay(const void* A, const void* B, void* out, int M, int N, int K, int lda, int ldb, int ldo,
                                  int bf16_out, const void* w, float decay, void* decay_part, void* stream_) {
  using namespace dm;
  if (w == nullptr || decay_part == nullptr || M < 1 || N < 1 || K < 1) return -1;
  if ((lda & 7) || (ldb & 7)) return -3;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_2d_bf16(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, 64, 128);
  if (rc) return 100 + rc;
  rc = make_tmap_2d_bf16(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, 64, 128);
  if (rc) return 200 + rc;
  GemmParams p{M, N, (K + GEMM_BK - 1) / GEMM_BK, ldo, out, 0, nullptr, nullptr, nullptr,
               reinterpret_cast<const float*>(w), reinterpret_cast<double*>(decay_part), decay};
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (bf16_out) return launch_gemm<128, true, true, EPI_STORE_BF16_DECAY>(tmA, tmB, p, 1, stream);
  return launch_gemm<128, true, true, EPI_STORE_F32_DECAY>(tmA, tmB, p, 1, stream);
}

// fc1 dgrad fused with the maxpool2/ReLU2 backward, and the conv2 bias gradient's per-CTA partials:
//   dxfc[b, j] = sum_k dh[b, k] * W1[j, k]   (A = dh [B,512] K-major, B = W1 [3136,512] rows = j, K contiguous)
//   dy2[b, 2ph+dy, 2pw+dx, c] = dxfc[b, (ph*7+pw)*64 + c] where code says (dy,dx) is the argmax and ReLU was active
//   bias_part[cta][c] = the CTA's sum of the scattered values of channel c.      dy2: [B,14,14,64] bf16, fully written (zeros included).
// bias_part holds dm_unpool_bias_slots(B) slots of 64 floats.
extern "C" int dm_fc1_dgrad_unpool_slots(const void* dh, const void* w1_bf16, const void* code2, void* dy2, void* bias_part,
                                         int B, void* stream_) {
  using namespace dm;
  CUtensorMap tmA, tmB;
  int rc = make_tmap_2d_bf16(&tmA, dh, 512, (uint64_t)B, 512, 64, 128, 128);
  if (rc) return 100 + rc;
  rc = make_tmap_2d_bf16(&tmB, w1_bf16, 512, 3136, 512, 64, 64, 128);
  if (rc) return 200 + rc;
  if (bias_part == nullptr) return -1;
  GemmParams p{B, 3136, 512 / GEMM_BK, 0, dy2, 0, nullptr, reinterpret_cast<const uint8_t*>(code2),
               reinterpret_cast<float*>(bias_part)};
  return launch_gemm<64, false, false, EPI_UNPOOL2_BF16>(tmA, tmB, p, 1, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int dm_unpool_bias_slots(int B) { return dm::unpool_bias_slots(B); }

// The same, with g_bias2[c] += the slots' sum in CTA order (pre-zeroed; bit-reproducible): the GEMM into a static
// workspace, then unpool_bias_sum.  Returns -6 without launching for a batch above the workspace's 10 624 rows.
extern "C" int dm_fc1_dgrad_unpool(const void* dh, const void* w1_bf16, const void* code2, void* dy2, void* g_bias2, int B,
                                   void* stream_) {
  using namespace dm;
  const int n = unpool_bias_slots(B);
  if (n > UNPOOL_MAX_CTAS) return -6;
  float* slots = nullptr;
  DM_CUDA_OK(cudaGetSymbolAddress(reinterpret_cast<void**>(&slots), g_unpool_bias_part));
  const int rc = dm_fc1_dgrad_unpool_slots(dh, w1_bf16, code2, dy2, slots, B, stream_);
  if (rc) return rc;
  return (int)launch_kernel(unpool_bias_sum_kernel, dim3(16), dim3(64), 0, reinterpret_cast<cudaStream_t>(stream_),
                            static_cast<const float*>(slots), n, reinterpret_cast<float*>(g_bias2));
}
