// conv1 (5x5 SAME, 1 -> 32 channels, 28x28 images) on the tensor cores: forward and weight gradient.
// reference ops K1-K4 (tf.nn.conv2d #1 + bias + ReLU + max_pool, src/mnist.py:107-118) and their gradients.
//
// K = 25 taps is too thin to be FLOP-relevant, but SIMT kernels sit on the fp32 FMA-pipe floor, so the thin
// GEMMs move to wgmma anyway.  With C_in = 1 no TMA box can express the im2col operand (a K
// step would be 2 bytes), so the operands are built in shared memory by software, in the swizzled layouts TMA would
// write.
//
//   forward  Tile = 128 consecutive POOLED pixels (flat index over batch x 14 x 14).  For each of the four positions p
//            of the 2x2 pooling window there is one im2col tile  A_p[128 pooled pixels][32 taps]  (taps 0-24 = the 5x5
//            window of conv pixel (2ph + p/2, 2pw + p%2), tap 25 = 1.0, taps 26-31 = 0; 64-byte swizzle), read
//            row-wise with ldmatrix.  D_p[pixel, co] = A_p * W[tap, co]: four m64n32 accumulators per warpgroup; every
//            thread holds the same (pixel, channel) positions of all four, so the 2x2 max-pool is an in-thread max,
//            fused with bias, ReLU and the argmax code.
//   wgrad    One row per pooled pixel P = (b, ph, pw): its 6x6 input patch X_P (input rows 2ph-2 .. 2ph+3, columns
//            2pw-2 .. 2pw+3), element j = 6 r + c, then a 1.0 at j = 36 (0 for padding pixels past the batch), then
//            zeros up to 64 bf16 = 128 B (128-byte swizzle).  The 5x5 window of position p = (dy, dx) lies inside the
//            patch: tap (kh, kw) of position p is X_P[(dy + kh) 6 + dx + kw].  E[j, (p, co)] = sum_P X_P[j] G_P[p, co]
//            with the patch tile read MN-major as A (M = j) and N = 128 = (p, co), where G_P keeps a pooled gradient
//            only where the forward pass selected position p and ReLU was active (pool/ReLU backward fused into the
//            operand build).  Each CTA folds E to dW[kh, kw, co] = sum_p E[(dy + kh) 6 + dx + kw, 32 p + co] and
//            db[co] = sum_p E[36, 32 p + co] (p in order 0..3), and the CTAs' partial sums are added up in a fixed
//            order, so the gradient is the same to the bit in every run.
#include "common.cuh"
#include "host_utils.h"

namespace dm {

constexpr int C1T_FW_THREADS = 256;       // two warpgroups: operand builders, then MMA + epilogue
constexpr int C1T_TILE = 128;             // pooled pixels per tile
constexpr int C1T_AP_BYTES = 128 * 64;    // one A_p tile: 128 rows x 32 bf16
constexpr int C1T_ROW_BYTES = 128;        // one patch row of the weight gradient: 64 bf16

struct ZeroRanges3 {
  float* ptr[3];
  int n[3];
};

// 16-byte chunk `c` of 64-byte row `r` inside a 64B-swizzled tile (address bits [4,5] ^= bits [7,8])
DMNIST_DEVICE uint32_t swz64(uint32_t r, uint32_t c) { return r * 64u + ((c ^ ((r >> 1) & 3u)) << 4); }
// 16-byte chunk `c` of 128-byte row `r` inside a 128B-swizzled, 1024-aligned tile (address bits [4,7) ^= bits [7,10))
DMNIST_DEVICE uint32_t swz128(uint32_t r, uint32_t c) { return r * 128u + ((c ^ (r & 7u)) << 4); }

DMNIST_DEVICE void sts128(uint8_t* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  *reinterpret_cast<uint4*>(p) = make_uint4(a, b, c, d);
}

// The im2col rows of pooled pixel P (thread = row m of the tile) for window positions p = 2h, 2h+1 (conv row 2ph + h)
// go to A_{2h}, A_{2h+1}.  Two threads share a pooled pixel, one per h, so a tile has 256 builders.  Loading and
// packing are separate steps: the loop prefetches the next tile's patch (global loads in flight) while it packs and
// stores the current one, so a builder pays the load latency once per CTA instead of once per tile.
struct PatchRegs {
  float v[5][6];        // input rows 2ph-2+h .. 2ph+2+h, columns 2pw-2 .. 2pw+3
  float one;            // 1.0 for real pixels (tap 25 = bias / ones column), 0 for padding rows of the last tile
};

DMNIST_DEVICE void load_patch_half(PatchRegs& pr, int h, long long P, long long total, const float* __restrict__ images) {
  if (P < total) {
    const int b = (int)(P / 196), pos = (int)(P - (long long)b * 196);
    const int ph = pos / 14, pw = pos - ph * 14;
    const float* img = images + (size_t)b * 784;
#pragma unroll
    for (int r = 0; r < 5; ++r) {
      const int y = 2 * ph - 2 + h + r;
#pragma unroll
      for (int c2 = 0; c2 < 3; ++c2) {
        const int x = 2 * pw - 2 + 2 * c2;           // even: the pair (x, x+1) is inside or outside as a whole
        float2 v = make_float2(0.f, 0.f);
        if (y >= 0 && y < 28 && x >= 0 && x < 28) v = __ldg(reinterpret_cast<const float2*>(img + y * 28 + x));
        pr.v[r][2 * c2] = v.x;
        pr.v[r][2 * c2 + 1] = v.y;
      }
    }
    pr.one = 1.f;
  } else {
#pragma unroll
    for (int r = 0; r < 5; ++r)
#pragma unroll
      for (int c = 0; c < 6; ++c) pr.v[r][c] = 0.f;
    pr.one = 0.f;
  }
}

DMNIST_DEVICE void store_im2col_half(uint8_t* a_tiles, int m, int h, const PatchRegs& pr) {
#pragma unroll
  for (int px = 0; px < 2; ++px) {
    uint32_t w[16];                                   // 32 taps as bf16 pairs
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int t0 = 2 * j, t1 = 2 * j + 1;
      const float v0 = t0 < 25 ? pr.v[t0 / 5][px + t0 % 5] : (t0 == 25 ? pr.one : 0.f);
      const float v1 = t1 < 25 ? pr.v[t1 / 5][px + t1 % 5] : (t1 == 25 ? pr.one : 0.f);
      w[j] = pack_bf16x2(v0, v1);
    }
    uint8_t* tile = a_tiles + (2 * h + px) * C1T_AP_BYTES;
#pragma unroll
    for (int c = 0; c < 4; ++c) sts128(tile + swz64(m, c), w[4 * c], w[4 * c + 1], w[4 * c + 2], w[4 * c + 3]);
  }
}

// ------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------
struct C1FwSmem {
  static constexpr int W_OFF = 0;                               // W[32 taps][32 co] bf16, MN-major, 64B swizzle (2 KB)
  static constexpr int A_OFF = 2048;                            // 2 stages x 4 x 8 KB
  static constexpr int BIAS_OFF = A_OFF + 2 * 4 * C1T_AP_BYTES; // 32 floats
  static constexpr int TOTAL = BIAS_OFF + 128 + 1024;
};

// Thread = builder of half a pooled pixel's im2col rows (pixel m = tid % 128, window row h = tid / 128), then one of
// the 256 MMA / epilogue threads.  Two operand stages: one __syncthreads per tile.
__global__ void __launch_bounds__(C1T_FW_THREADS, 1)
conv1_fwd_tc_kernel(const float* __restrict__ images,   // [B,28,28] fp32
                    const float* __restrict__ w,        // [25][32] fp32
                    const float* __restrict__ bias,     // [32]
                    __nv_bfloat16* __restrict__ out,    // [B,14,14,32]
                    uint8_t* __restrict__ code,         // [B,14,14,32]
                    long long total,                    // B * 196 pooled pixels
                    int num_tiles, ZeroRanges3 zr) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* s_bias = reinterpret_cast<float*>(smem + C1FwSmem::BIAS_OFF);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x < 32) s_bias[lane] = __ldg(bias + lane);
  if (threadIdx.x < 128) {
    // weights: fp32 [25][32] -> bf16 rows of 64 B (k-row = tap), rows 25-31 zero.  128 threads x one 16-byte chunk.
    const int k = threadIdx.x >> 2, c = threadIdx.x & 3;
    uint32_t pk[4] = {0u, 0u, 0u, 0u};
    if (k < 25) {
      const float4 lo = __ldg(reinterpret_cast<const float4*>(w + k * 32 + c * 8));
      const float4 hi = __ldg(reinterpret_cast<const float4*>(w + k * 32 + c * 8 + 4));
      pk[0] = pack_bf16x2(lo.x, lo.y); pk[1] = pack_bf16x2(lo.z, lo.w);
      pk[2] = pack_bf16x2(hi.x, hi.y); pk[3] = pack_bf16x2(hi.z, hi.w);
    }
    sts128(smem + C1FwSmem::W_OFF + swz64(k, c), pk[0], pk[1], pk[2], pk[3]);
  }
  fence_proxy_async_smem();                       // W is read by wgmma (async proxy)
  __syncthreads();
  pdl_wait();
  // first kernel of a training step: clear the atomically accumulated gradient regions and the loss accumulator
  {
    const int gi = blockIdx.x * C1T_FW_THREADS + threadIdx.x;
#pragma unroll
    for (int r = 0; r < 3; ++r)
      if (zr.ptr[r] != nullptr)
        for (int i = gi; i < zr.n[r]; i += gridDim.x * C1T_FW_THREADS) zr.ptr[r][i] = 0.f;
  }

  const int h = threadIdx.x >> 7, m = threadIdx.x & 127;         // builder role
  // W as B (MN-major, 64B swizzle): k-row = tap (64 B = 32 co), 8-row groups 512 B apart; K step of 16 taps = 1024 B
  const uint64_t db0 = make_smem_desc(smem_u32(smem + C1FwSmem::W_OFF), 8192, 512, SWZ_64B);
  // ldmatrix rows of this lane: x4 tiles 0/1 = rows +0 / +8, tiles 2/3 = taps + 8
  const int lr = 16 * warp + (lane & 7) + ((lane >> 3) & 1) * 8, kc = lane >> 4;
  PatchRegs cur, nxt;
  load_patch_half(cur, h, (long long)blockIdx.x * C1T_TILE + m, total, images);
  float acc[4][16];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[p][j] = 0.f;
  int i = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++i) {
    const int s = i & 1;
    const int tn = t + gridDim.x;
    if (tn < num_tiles) load_patch_half(nxt, h, (long long)tn * C1T_TILE + m, total, images);   // in flight during the stores
    uint8_t* stage = smem + C1FwSmem::A_OFF + s * 4 * C1T_AP_BYTES;
    store_im2col_half(stage, m, h, cur);
    __syncthreads();     // stage s complete; every thread is past its reads of stage s ^ 1 (written next iteration)

    uint32_t a[4][2][4];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int k = 0; k < 2; ++k) ldsm_x4(smem_u32(stage + p * C1T_AP_BYTES + swz64(lr, 2 * k + kc)), a[p][k]);
#pragma unroll
    for (int p = 0; p < 4; ++p) fence_regs(acc[p]);
    wgmma_fence();
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int k = 0; k < 2; ++k) wgmma_m64n32_rs<1>(acc[p], a[p][k], desc_advance(db0, 1024 * k), k);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int p = 0; p < 4; ++p) fence_regs(acc[p]);

    // epilogue: max-pool over the four accumulators in registers, bias, ReLU, argmax code
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const long long P = (long long)t * C1T_TILE + 16 * warp + (lane >> 2) + 8 * half;
      if (P >= total) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        float o[2];
        uint32_t cd = 0u;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int ai = 4 * j + 2 * half + e;
          float mx = acc[0][ai];
          uint32_t idx = 0;
#pragma unroll
          for (int p = 1; p < 4; ++p)
            if (acc[p][ai] > mx) { mx = acc[p][ai]; idx = p; }
          mx += s_bias[col + e];
          const bool active = mx > 0.f;
          cd |= (idx | (active ? 4u : 0u)) << (8 * e);
          o[e] = active ? mx : 0.f;
        }
        const size_t off = (size_t)P * 32 + col;
        *reinterpret_cast<uint32_t*>(out + off) = pack_bf16x2(o[0], o[1]);
        *reinterpret_cast<uint16_t*>(code + off) = (uint16_t)cd;
      }
    }
    cur = nxt;
  }
}

// Two threads build a patch row: half h = 0 writes chunks 0-3 (j 0..31), half h = 1 chunks 4-7 (j 32..35, the 1.0 and
// zeros).  Loading and packing are separate steps, so the loads of the next tile are in flight while the current tile
// is multiplied.
template <int H>
DMNIST_DEVICE void load_patch_row_half_t(float (&v)[32], long long P, long long total, const float* __restrict__ images) {
  if (P < total) {
    const int b = (int)(P / 196), pos = (int)(P - (long long)b * 196);
    const int ph = pos / 14, pw = pos - ph * 14;
    const float* img = images + (size_t)b * 784;
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int j = 32 * H + 2 * u;
      if (j < 36) {
        const int y = 2 * ph - 2 + j / 6, x = 2 * pw - 2 + j % 6;   // x even: the pair (x, x+1) is inside or outside as a whole
        float2 t = make_float2(0.f, 0.f);
        if (y >= 0 && y < 28 && x >= 0 && x < 28) t = __ldg(reinterpret_cast<const float2*>(img + y * 28 + x));
        v[2 * u] = t.x;
        v[2 * u + 1] = t.y;
      } else {
        v[2 * u] = j == 36 ? 1.f : 0.f;
        v[2 * u + 1] = 0.f;
      }
    }
  } else {
#pragma unroll
    for (int u = 0; u < 32; ++u) v[u] = 0.f;
  }
}

DMNIST_DEVICE void load_patch_row_half(float (&v)[32], int h, long long P, long long total, const float* __restrict__ images) {
  if (h == 0) load_patch_row_half_t<0>(v, P, total, images);
  else load_patch_row_half_t<1>(v, P, total, images);
}

DMNIST_DEVICE void store_patch_row_half(uint8_t* tile, int m, int h, const float (&v)[32]) {
#pragma unroll
  for (int c = 0; c < 4; ++c)
    sts128(tile + swz128(m, 4 * h + c), pack_bf16x2(v[8 * c], v[8 * c + 1]), pack_bf16x2(v[8 * c + 2], v[8 * c + 3]),
           pack_bf16x2(v[8 * c + 4], v[8 * c + 5]), pack_bf16x2(v[8 * c + 6], v[8 * c + 7]));
}

// ------------------------------------------------------------------------------------------------------
// weight gradient (+ bias gradient from the 1.0 at j = 36), fused with the maxpool1 / ReLU1 backward
// ------------------------------------------------------------------------------------------------------
// One warpgroup per CTA over a contiguous range of 64-pixel tiles.  Thread (m, h) builds half h of pixel m's patch row
// and G half h: the masked gradient of positions 2h, 2h+1 (128 B).  A three-stage ring with one barrier per stage and
// one commit group per tile, waited with wait_group 1: the builders fill the next stage while the tensor core works on
// this one.  The stage written at tile i was last read by tile i - 3's MMAs, which every warp has waited for before the
// barrier of tile i - 1.
constexpr int C1WG_THREADS = 128;
constexpr int C1WG_TILE = 64;
constexpr int C1WG_STAGES = 3;
constexpr int C1WG_SLOT = 26 * 32;        // taps 0-24, then the bias
constexpr int C1WG_MAX_SLOTS = 512;
constexpr int C1WG_MAX_GROUPS = 32;       // >= ceil(sqrt(C1WG_MAX_SLOTS))
// Two-level reduction of the per-CTA slots: the last CTA of each group of `group` consecutive CTAs adds its group's
// slots in slot order into a group slot, the last group to finish adds the group slots in order into g_w / g_b.  One
// launch of this kernel in flight per device: the workspaces and tickets are static (see arrive_last_cta).
static_assert(C1WG_MAX_GROUPS * C1WG_MAX_GROUPS >= C1WG_MAX_SLOTS, "too few group slots");
__device__ __align__(16) float g_c1wg_part[C1WG_MAX_SLOTS * C1WG_SLOT];
__device__ __align__(16) float g_c1wg_group[C1WG_MAX_GROUPS * C1WG_SLOT];
__device__ unsigned int g_c1wg_group_ticket[C1WG_MAX_GROUPS];
__device__ unsigned int g_c1wg_ticket;

struct C1WgSmem {
  static constexpr int PATCH_BYTES = C1WG_TILE * C1T_ROW_BYTES;  // [64 pixels][64 j] bf16
  static constexpr int G_BYTES = 2 * C1WG_TILE * 128;            // two [64 pixels][64 (p, co)] bf16 halves
  static constexpr int STAGE_BYTES = PATCH_BYTES + G_BYTES;
  static constexpr int E_LD = 136;                               // fold scratch: E rows 0..36, fp32, over the ring
  static constexpr int TOTAL = C1WG_STAGES * STAGE_BYTES + 1024;
  static_assert(37 * E_LD * 4 <= C1WG_STAGES * STAGE_BYTES, "fold scratch exceeds the ring");
};

__global__ void __launch_bounds__(C1WG_THREADS, 1)
conv1_wgrad_tc_kernel(const float* __restrict__ images,          // [B,28,28]
                      const __nv_bfloat16* __restrict__ dpool,   // [B,14,14,32] gradient w.r.t. the pooled activations
                      const uint8_t* __restrict__ code,          // [B,14,14,32]
                      float* __restrict__ g_w,                   // [25][32], the CTAs' sum is added to it (pre-zeroed)
                      float* __restrict__ g_b,                   // [32]
                      long long total, int num_tiles, int group) {
  using S = C1WgSmem;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // contiguous tile range per CTA
  const int t_begin = (int)(((long long)num_tiles * blockIdx.x) / gridDim.x);
  const int t_end = (int)(((long long)num_tiles * (blockIdx.x + 1)) / gridDim.x);
  const int nt = t_end - t_begin;
  pdl_wait();

  const int h = threadIdx.x / C1WG_TILE, m = threadIdx.x % C1WG_TILE;     // builder role
  float v[32];
  uint4 gq[4];      // pooled gradient, 32 channels bf16
  uint4 cq[2];      // pooling codes, 32 channels
  auto load_tile = [&](int i) {
    const long long P = (long long)(t_begin + i) * C1WG_TILE + m;
    load_patch_row_half(v, h, P, total, images);
    if (P < total) {
      const uint4* gp = reinterpret_cast<const uint4*>(dpool + (size_t)P * 32);
      const uint4* cp = reinterpret_cast<const uint4*>(code + (size_t)P * 32);
#pragma unroll
      for (int j = 0; j < 4; ++j) gq[j] = gp[j];
      cq[0] = __ldg(cp);
      cq[1] = __ldg(cp + 1);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) gq[j] = make_uint4(0, 0, 0, 0);
      cq[0] = cq[1] = make_uint4(0, 0, 0, 0);
    }
  };
  float acc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0.f;
  if (nt > 0) load_tile(0);
  for (int i = 0; i < nt; ++i) {
    uint8_t* stage = smem + (i % C1WG_STAGES) * S::STAGE_BYTES;
    store_patch_row_half(stage, m, h, v);
    const uint32_t g32[16] = {gq[0].x, gq[0].y, gq[0].z, gq[0].w, gq[1].x, gq[1].y, gq[1].z, gq[1].w,
                              gq[2].x, gq[2].y, gq[2].z, gq[2].w, gq[3].x, gq[3].y, gq[3].z, gq[3].w};
    const uint32_t cw[8] = {cq[0].x, cq[0].y, cq[0].z, cq[0].w, cq[1].x, cq[1].y, cq[1].z, cq[1].w};
    uint8_t* g_half = stage + S::PATCH_BYTES + h * (C1WG_TILE * 128);
#pragma unroll
    for (int px = 0; px < 2; ++px) {
      const uint32_t p = 2u * (uint32_t)h + (uint32_t)px;
      uint32_t o[16];
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) {     // same byte-parallel mask as the unpool epilogue of gemm_tc.cu
        const uint32_t xz = (cw[w8] & 0x07070707u) ^ (0x04040404u | (0x01010101u * p));
        const uint32_t hit = ~(xz + 0x7f7f7f7fu) & 0x80808080u;
        o[2 * w8] = g32[2 * w8] & prmt(hit, 0u, 0x9988u);
        o[2 * w8 + 1] = g32[2 * w8 + 1] & prmt(hit, 0u, 0xbbaau);
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) sts128(g_half + swz128(m, 4 * px + c), o[4 * c], o[4 * c + 1], o[4 * c + 2], o[4 * c + 3]);
    }
    if (i + 1 < nt) load_tile(i + 1);             // in flight during the MMAs
    fence_proxy_async_smem();                     // the operands are read by wgmma (async proxy)
    __syncthreads();

    // A = patch rows read MN-major (M = j, one 128 B chunk), B = G MN-major (N = 128: two chunks 8 KB apart); both
    // with pixel k-rows of 128 B, 8-row groups 1024 B apart: a K step of 16 pixels is 2048 B
    const uint64_t da = make_smem_desc(smem_u32(stage), 8192, 1024, SWZ_128B);
    const uint64_t db = make_smem_desc(smem_u32(stage + S::PATCH_BYTES), 8192, 1024, SWZ_128B);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n128_ss<1, 1>(acc, desc_advance(da, 2048 * ks), desc_advance(db, 2048 * ks), 1);
    wgmma_commit();
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  fence_regs(acc);
  __syncthreads();                                // every warp's MMAs are done with the ring: the fold scratch reuses it

  // E rows 0..36 -> shared memory, then fold the four positions into this CTA's slot
  float* E = reinterpret_cast<float*>(smem);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int r = 16 * warp + (lane >> 2) + 8 * half;
    if (r < 37) {
#pragma unroll
      for (int j = 0; j < 16; ++j)
        *reinterpret_cast<float2*>(E + r * S::E_LD + 8 * j + 2 * (lane & 3)) = make_float2(acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
    }
  }
  __syncthreads();
  float* part = g_c1wg_part + (size_t)blockIdx.x * C1WG_SLOT;
  for (int e = threadIdx.x; e < C1WG_SLOT; e += C1WG_THREADS) {
    const int tap = e >> 5, co = e & 31;
    float s = 0.f;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int j = tap < 25 ? ((p >> 1) + tap / 5) * 6 + (p & 1) + tap % 5 : 36;
      s += E[j * S::E_LD + 32 * p + co];
    }
    part[e] = s;
  }

  __shared__ unsigned int s_last;
  const int grp = blockIdx.x / group, g0 = grp * group;
  const int gn = min(group, (int)gridDim.x - g0), ngroups = ((int)gridDim.x + group - 1) / group;
  if (!arrive_last_cta(&g_c1wg_group_ticket[grp], gn, 1, C1WG_THREADS, &s_last)) return;
  float4* gslot = reinterpret_cast<float4*>(g_c1wg_group + (size_t)grp * C1WG_SLOT);
  for (int e4 = threadIdx.x; e4 < C1WG_SLOT / 4; e4 += C1WG_THREADS)
    gslot[e4] = ordered_sum4(reinterpret_cast<const float4*>(g_c1wg_part + (size_t)g0 * C1WG_SLOT) + e4, gn, C1WG_SLOT / 4);
  if (!arrive_last_cta(&g_c1wg_ticket, ngroups, 1, C1WG_THREADS, &s_last)) return;
  for (int e4 = threadIdx.x; e4 < C1WG_SLOT / 4; e4 += C1WG_THREADS) {
    const float4 sum = ordered_sum4(reinterpret_cast<const float4*>(g_c1wg_group) + e4, ngroups, C1WG_SLOT / 4);
    const int row = e4 >> 3, col = (e4 & 7) * 4;
    float4* o = reinterpret_cast<float4*>((row < 25 ? g_w + row * 32 : g_b) + col);
    const float4 cur = *o;
    *o = make_float4(cur.x + sum.x, cur.y + sum.y, cur.z + sum.z, cur.w + sum.w);
  }
}

}  // namespace dm

extern "C" {

int dm_conv1_fwd_tc(const void* images, const void* w, const void* bias, void* out, void* code, int B, void* zero0,
                    int n0, void* zero1, int n1, void* zero2, int n2, void* stream) {
  using namespace dm;
  ZeroRanges3 zr;
  zr.ptr[0] = reinterpret_cast<float*>(zero0); zr.n[0] = n0;
  zr.ptr[1] = reinterpret_cast<float*>(zero1); zr.n[1] = n1;
  zr.ptr[2] = reinterpret_cast<float*>(zero2); zr.n[2] = n2;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(conv1_fwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C1FwSmem::TOTAL));
    DM_CUDA_OK(cudaFuncSetAttribute(conv1_fwd_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  const long long total = (long long)B * 196;
  const int tiles = (int)((total + C1T_TILE - 1) / C1T_TILE);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  return (int)launch_kernel(conv1_fwd_tc_kernel, dim3(grid), dim3(C1T_FW_THREADS), C1FwSmem::TOTAL,
                            reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const float*>(images),
                            reinterpret_cast<const float*>(w), reinterpret_cast<const float*>(bias),
                            reinterpret_cast<__nv_bfloat16*>(out), reinterpret_cast<uint8_t*>(code), total, tiles, zr);
}

}  // extern "C"

// g_w [25][32] and g_b [32] must be zeroed by the caller (the gradient is added to them).
extern "C" int dm_conv1_wgrad_tc(const void* images, const void* dpool, const void* code, void* g_w, void* g_b, int B, void* stream) {
  using namespace dm;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(conv1_wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C1WgSmem::TOTAL));
    DM_CUDA_OK(cudaFuncSetAttribute(conv1_wgrad_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  const long long total = (long long)B * 196;
  const int tiles = (int)((total + C1WG_TILE - 1) / C1WG_TILE);
  int grid = tiles < max_ctas() ? tiles : max_ctas();
  if (grid > C1WG_MAX_SLOTS) grid = C1WG_MAX_SLOTS;
  int group = 1;                                  // ceil(sqrt(grid)) CTAs per group, so at most as many groups
  while (group * group < grid) ++group;
  return (int)launch_kernel(conv1_wgrad_tc_kernel, dim3(grid), dim3(C1WG_THREADS), C1WgSmem::TOTAL,
                            reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const float*>(images),
                            reinterpret_cast<const __nv_bfloat16*>(dpool), reinterpret_cast<const uint8_t*>(code),
                            reinterpret_cast<float*>(g_w), reinterpret_cast<float*>(g_b), total, tiles, group);
}
