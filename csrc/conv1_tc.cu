// conv1 (5x5 SAME, 1 -> 32 channels, 28x28 images) on the tensor cores: forward and weight gradient.
// reference ops K1-K4 (tf.nn.conv2d #1 + bias + ReLU + max_pool, src/mnist.py:107-118) and their gradients.
//
// K = 25 taps is too thin to be FLOP-relevant, but SIMT kernels sit on the fp32 FMA-pipe floor, so the thin
// GEMMs move to wgmma anyway.  With C_in = 1 no TMA box can express the im2col operand (a K
// step would be 2 bytes), so the operand is built in shared memory by software -- 36 input values per pooled
// pixel -- in the 64-byte-swizzled layout TMA would write.
//
// Tile = 128 consecutive POOLED pixels (flat index over batch x 14 x 14).  For each of the four positions p of the
// 2x2 pooling window there is one im2col tile  A_p[128 pooled pixels][32 taps]  (taps 0-24 = the 5x5 window of conv
// pixel (2ph + p/2, 2pw + p%2), tap 25 = 1.0, taps 26-31 = 0).  Read row-wise (ldmatrix) it is the forward A
// (rows = M = pixels, K = taps); read transposed (ldmatrix.trans) it is the weight-gradient A (M = taps,
// K = pixels): same bytes.
//
//   forward  D_p[pixel, co] = A_p * W[tap, co]   four m64n32 accumulators per warpgroup; every thread holds the
//            same (pixel, channel) positions of all four, so the 2x2 max-pool is an in-thread max, fused with
//            bias, ReLU and the argmax code.
//   wgrad    D[tap, co] += A_p^T * G_p[pixel, co]   where G_p keeps a pooled gradient only where the forward pass
//            selected position p and ReLU was active (pool/ReLU backward fused into the operand build); tap 25
//            accumulates the bias gradient.  Accumulators stay in registers for the CTA's whole pixel range; the
//            CTAs' partial sums are added up in a fixed order, so the gradient is the same to the bit in every run.
#include "common.cuh"
#include "host_utils.h"

namespace dm {

constexpr int C1T_FW_THREADS = 256;       // two warpgroups: operand builders, then MMA + epilogue
constexpr int C1T_TILE = 128;             // pooled pixels per tile
constexpr int C1T_AP_BYTES = 128 * 64;    // one A_p (or G_p) tile: 128 rows x 32 bf16

struct ZeroRanges3 {
  float* ptr[3];
  int n[3];
};

// 16-byte chunk `c` of 64-byte row `r` inside a 64B-swizzled tile (address bits [4,5] ^= bits [7,8])
DMNIST_DEVICE uint32_t swz64(uint32_t r, uint32_t c) { return r * 64u + ((c ^ ((r >> 1) & 3u)) << 4); }

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

DMNIST_DEVICE void store_im2col_half(uint8_t* a_tiles, int m, int h, const PatchRegs& pr, int tile_bytes = C1T_AP_BYTES) {
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
    uint8_t* tile = a_tiles + (2 * h + px) * tile_bytes;
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

// ------------------------------------------------------------------------------------------------------
// weight gradient (+ bias gradient as tap 25), fused with the maxpool1 / ReLU1 backward
// ------------------------------------------------------------------------------------------------------
// TILE = 64 or 128 pooled pixels per tile; 2 * TILE threads (two builders per pooled pixel: window rows h = 0, 1) =
// TILE / 64 warpgroups, warpgroup g reducing over pixels 64 g .. 64 g + 63 of every tile.  M = 64 rows of taps of
// which 32 are real: warps 2 and 3 of a warpgroup feed zero operands.  The 64-pixel tile needs half the shared
// memory (2 x 32 KB), so a CTA fits next to conv2_wgrad's and the two weight-gradient kernels can overlap.
// Per-warpgroup partial sums of the weight gradient (rows = taps, 25 = bias; rows 26-31 unused), reduced in slot order
// by the last CTA (see arrive_last_cta).
constexpr int C1WG_SLOT = 32 * 32;
constexpr int C1WG_MAX_SLOTS = 512;
// One launch of this kernel in flight per device: the workspace and ticket are static (see arrive_last_cta).
__device__ float g_c1wg_part[C1WG_MAX_SLOTS * C1WG_SLOT];
__device__ unsigned int g_c1wg_ticket;

template <int TILE>
struct C1WgSmem {
  static constexpr int TILE_BYTES = TILE * 64;                   // TILE pooled pixels x 32 bf16
  static constexpr int STAGE_BYTES = 8 * TILE_BYTES;            // A_0..A_3 then G_0..G_3
  static constexpr int TOTAL = 2 * STAGE_BYTES + 1024;
};

template <int TILE>
__global__ void __launch_bounds__(2 * TILE, 1)
conv1_wgrad_tc_kernel(const float* __restrict__ images,          // [B,28,28]
                      const __nv_bfloat16* __restrict__ dpool,   // [B,14,14,32] gradient w.r.t. the pooled activations
                      const uint8_t* __restrict__ code,          // [B,14,14,32]
                      float* __restrict__ g_w,                   // [25][32], the CTAs' sum is added to it (pre-zeroed)
                      float* __restrict__ g_b,                   // [32]
                      long long total, int num_tiles) {
  using S = C1WgSmem<TILE>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // contiguous tile range per CTA
  const int t_begin = (int)(((long long)num_tiles * blockIdx.x) / gridDim.x);
  const int t_end = (int)(((long long)num_tiles * (blockIdx.x + 1)) / gridDim.x);
  const int nt = t_end - t_begin;
  pdl_wait();

  const int h = threadIdx.x / TILE, m = threadIdx.x % TILE;     // builder role
  const int wg = warp >> 2, wq = warp & 3;                       // MMA role: warpgroup, warp inside it
  // A_p^T via ldmatrix.trans: x4 tile i covers taps + 8 (i & 1) and pixels + 8 (i >> 1)
  const int a_chunk = 2 * wq + ((lane >> 3) & 1);
  const int a_row = 64 * wg + 8 * (lane >> 4) + (lane & 7);
  struct TileRegs {
    PatchRegs patch;
    uint4 gq[4];      // pooled gradient, 32 channels bf16
    uint4 cq[2];      // pooling codes, 32 channels
  };
  auto load_tile = [&](TileRegs& tr, int i) {
    const long long P = (long long)(t_begin + i) * TILE + m;
    load_patch_half(tr.patch, h, P, total, images);
    if (P < total) {
      const uint4* gp = reinterpret_cast<const uint4*>(dpool + (size_t)P * 32);
      const uint4* cp = reinterpret_cast<const uint4*>(code + (size_t)P * 32);
#pragma unroll
      for (int j = 0; j < 4; ++j) tr.gq[j] = gp[j];
      tr.cq[0] = __ldg(cp);
      tr.cq[1] = __ldg(cp + 1);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) tr.gq[j] = make_uint4(0, 0, 0, 0);
      tr.cq[0] = tr.cq[1] = make_uint4(0, 0, 0, 0);
    }
  };
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  TileRegs cur, nxt;
  if (nt > 0) load_tile(cur, 0);
  for (int i = 0; i < nt; ++i) {
    const int s = i & 1;
    uint8_t* stage = smem + s * S::STAGE_BYTES;
    if (i + 1 < nt) load_tile(nxt, i + 1);        // next tile's global loads are in flight while this one is packed
    store_im2col_half(stage, m, h, cur.patch, S::TILE_BYTES);
    const uint4* gq = cur.gq;
    const uint4* cq = cur.cq;
    const uint32_t g32[16] = {gq[0].x, gq[0].y, gq[0].z, gq[0].w, gq[1].x, gq[1].y, gq[1].z, gq[1].w,
                              gq[2].x, gq[2].y, gq[2].z, gq[2].w, gq[3].x, gq[3].y, gq[3].z, gq[3].w};
    const uint32_t cw[8] = {cq[0].x, cq[0].y, cq[0].z, cq[0].w, cq[1].x, cq[1].y, cq[1].z, cq[1].w};
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
      uint8_t* tile = stage + (4 + p) * S::TILE_BYTES;
#pragma unroll
      for (int c = 0; c < 4; ++c) sts128(tile + swz64(m, c), o[4 * c], o[4 * c + 1], o[4 * c + 2], o[4 * c + 3]);
    }
    fence_proxy_async_smem();                     // G_p is read by wgmma (async proxy)
    __syncthreads();     // stage s complete; every thread is past its reads of stage s ^ 1 (written next iteration)

    fence_regs(acc);
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      // G_p as B (MN-major, 64B swizzle): k-row = pooled pixel (64 B = 32 co), 8-row groups 512 B apart
      const uint32_t g_base = smem_u32(stage + (4 + p) * S::TILE_BYTES) + 64 * 64 * wg;
      uint32_t a[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        if (wq < 2) {
          ldsm_x4_trans(smem_u32(stage + p * S::TILE_BYTES + swz64(a_row + 16 * ks, a_chunk)), a[ks]);
        } else {
          a[ks][0] = a[ks][1] = a[ks][2] = a[ks][3] = 0u;
        }
      }
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        wgmma_m64n32_rs<1>(acc, a[ks], make_smem_desc(g_base + 1024 * ks, 8192, 512, SWZ_64B), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc);
    cur = nxt;
  }
  constexpr int NWG = TILE / 64;
  if (wq < 2) {
    // accumulator rows = taps (25 = bias) -> this warpgroup's slot
    float* part = g_c1wg_part + (size_t)(blockIdx.x * NWG + wg) * C1WG_SLOT;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int tap = 16 * wq + (lane >> 2) + 8 * half;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        *reinterpret_cast<float2*>(part + tap * 32 + 8 * j + 2 * (lane & 3)) =
            make_float2(acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
    }
  }
  __shared__ unsigned int s_last;
  if (arrive_last_cta(&g_c1wg_ticket, gridDim.x, 1, 2 * TILE, &s_last)) {
    const int nslots = gridDim.x * NWG;
    for (int e4 = threadIdx.x; e4 < 26 * 32 / 4; e4 += 2 * TILE) {
      const float4 sum = ordered_sum4(reinterpret_cast<const float4*>(g_c1wg_part) + e4, nslots, C1WG_SLOT / 4);
      const int row = e4 >> 3, col = (e4 & 7) * 4;
      float4* o = reinterpret_cast<float4*>((row < 25 ? g_w + row * 32 : g_b) + col);
      const float4 cur = *o;
      *o = make_float4(cur.x + sum.x, cur.y + sum.y, cur.z + sum.z, cur.w + sum.w);
    }
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

template <int TILE>
static int launch_conv1_wgrad(const void* images, const void* dpool, const void* code, void* g_w, void* g_b, int B,
                              void* stream) {
  using namespace dm;
  auto kern = conv1_wgrad_tc_kernel<TILE>;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C1WgSmem<TILE>::TOTAL));
    DM_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  const long long total = (long long)B * 196;
  const int tiles = (int)((total + TILE - 1) / TILE);
  int grid = tiles < max_ctas() ? tiles : max_ctas();
  if (grid * (TILE / 64) > C1WG_MAX_SLOTS) grid = C1WG_MAX_SLOTS / (TILE / 64);
  return (int)launch_kernel(kern, dim3(grid), dim3(2 * TILE), C1WgSmem<TILE>::TOTAL,
                            reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const float*>(images),
                            reinterpret_cast<const __nv_bfloat16*>(dpool), reinterpret_cast<const uint8_t*>(code),
                            reinterpret_cast<float*>(g_w), reinterpret_cast<float*>(g_b), total, tiles);
}

// g_w [25][32] and g_b [32] must be zeroed by the caller (the gradient is added to them).
extern "C" int dm_conv1_wgrad_tc(const void* images, const void* dpool, const void* code, void* g_w, void* g_b, int B, void* stream) {
  return launch_conv1_wgrad<64>(images, dpool, code, g_w, g_b, B, stream);
}
