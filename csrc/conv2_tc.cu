// conv2 (5x5 SAME, 32 -> 64 channels, 14x14 feature maps) as wgmma implicit GEMMs.
// reference op K5 (tf.nn.conv2d #2, src/mnist.py:119-122) = 82 % of the model FLOPs, fused with
// K2/K3/K4 (bias, ReLU, 2x2 max-pool, src/mnist.py:123-127) in the forward epilogue.
//
// No im2col buffer exists anywhere: activations stay NHWC bf16.  In fwd and dgrad an M tile is 128 real pixels of the
// batch: 32 consecutive pooled pixels x 4 window positions (fwd) or 128 consecutive pixels (dgrad), so a tile may span
// two images.  Seen as one stack of B * 14 image rows, its receptive field is at most 16 (fwd) or 14 (dgrad) consecutive
// full-width rows, staged by ONE TMA box (channels, 14 pixels, rows, 1) of fixed size per tile: 14 / 24.5 KB per stage.
// Taps whose source pixel lies outside the output pixel's own image (the SAME padding halo, or the neighbouring image in
// the stack) read a 1 KB zero block instead; a per-lane 25-bit mask, computed once per tile, picks them.
//
//   fwd    D[pixel, co]  += X[pixel + tap, ci] (A: registers)  * W[tap][ci][co] (B: MN-major smem, 128B swizzle)
//   dgrad  D[pixel, ci]  += dY[pixel - tap, co] (A: registers) * W[tap][ci][co] (B: K-major smem,  128B swizzle)
//   wgrad  D[(tap,ci), co] += X[pixel + tap, ci] (A: registers, transposed) * dY[pixel, co] (B: MN-major smem),
//          K = the pixels of whole images (an 18 x 18 patch and 208 dY rows per image), split over CTAs whose
//          partial sums a second kernel adds up in a fixed order (bit-reproducible).
// The A operand of every tap is the same patch shifted by (kh, kw): a window that starts at an arbitrary
// pixel of the swizzled patch, so each warp gathers its 16 rows with ldmatrix (addresses computed with the
// TMA swizzle) and hands them to wgmma in registers; B always starts on a swizzle-atom boundary and is
// read by wgmma straight from shared memory.  The HWIO bf16 weight image (800 x 64) is loaded once per
// CTA and stays resident in shared memory (100 KB) while the persistent CTA walks its tiles.
//
// Threads: warps 0-7 = two consumer warpgroups (rows 0-63 / 64-127 of a tile), warp 8 = TMA producer.
#include "common.cuh"
#include "host_utils.h"

namespace dm {

constexpr int CV_CONSUMERS = 256;
constexpr int CV_THREADS = CV_CONSUMERS + 32;
constexpr int W_BYTES = 800 * 64 * 2;   // 102400

// ldmatrix row address inside a patch of `row_bytes`-wide pixels written by TMA with a swizzle of the same width
// (64 B: 16-byte chunk bits [4,5] ^= address bits [7,8]; 128 B: bits [4,6] ^= bits [7,9]); patches start on a
// 1024-byte boundary.  Swizzling the full address (rather than adding a per-pixel swizzled offset to the base) leaves
// no loop-invariant per-tap offsets for the compiler to keep live across tiles; that keeps the pipelined tap loops at
// about 80 registers, so the fc1 update kernel's small CTAs still fit next to conv2_dgrad's in each SM sub-partition.
template <int ROW_BYTES>
DMNIST_DEVICE uint32_t patch_addr(uint32_t base, int pixel, int chunk) {
  const uint32_t a = base + pixel * ROW_BYTES + chunk * 16;
  return a ^ ((a >> 3) & (ROW_BYTES == 64 ? 0x30 : 0x70));
}

// Taps (bit kh * 5 + kw) whose source pixel (h + DIR * (kh - 2), w + DIR * (kw - 2)) lies inside the 14 x 14 image; the
// other taps read SAME padding.  Each coordinate's valid range of kh / kw is contiguous.
template <int DIR>
DMNIST_DEVICE uint32_t inside_taps(int h, int w) {
  const int rlo = max(0, DIR > 0 ? 2 - h : h - 11), rhi = min(4, DIR > 0 ? 15 - h : h + 2);
  const int clo = max(0, DIR > 0 ? 2 - w : w - 11), chi = min(4, DIR > 0 ? 15 - w : w + 2);
  const uint32_t rows = (1u << (5 * rhi + 5)) - (1u << (5 * rlo));   // every kw of kh in [rlo, rhi]
  const uint32_t cols = ((2u << chi) - (1u << clo)) * 0x108421u;      // kw in [clo, chi], repeated for each kh
  return rows & cols;
}

// ldmatrix row address of one tap: the staged pixel `pix`, or, for a tap that reads padding, pixel pix mod 8 of the
// zero block, so the eight rows of a matrix keep the distinct banks they would have had.
template <int ROW_BYTES>
DMNIST_DEVICE uint32_t tap_addr(uint32_t patch, uint32_t zero, uint32_t inside, int tap, int pix, int chunk) {
  const bool in = (inside >> tap) & 1;
  return patch_addr<ROW_BYTES>(in ? patch : zero, in ? pix : (pix & 7), chunk);
}

// First row of a tile's receptive field in the batch seen as one stack of B * 14 image rows: two rows above the tile's
// first pixel row, clipped at the top of its image.
DMNIST_DEVICE int first_staged_row(int stack_row) { return stack_row - min(stack_row % 14, 2); }

// ------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------
constexpr int FW_POOLED = 32;                  // pooled pixels per tile: 128 conv pixels = 32 x 4 window positions
constexpr int FW_ROWS = 16;                    // staged image rows per tile, the most any tile start needs
constexpr int FW_STAGES = 4;
constexpr int FW_A_BYTES = FW_ROWS * 14 * 32 * 2;   // 14 KB: 16 rows x 14 pixels x 32 ch
constexpr int FW_ACC_LD = 64 + 4;              // fp32 accumulator staging row (padded)
constexpr int ZERO_BYTES = 1024;               // 8 zero pixels of up to 128 B, read by the taps that fall in the padding
struct FwSmem {
  static constexpr int A_OFF = W_BYTES;
  static constexpr int ZERO_OFF = A_OFF + FW_STAGES * FW_A_BYTES;
  static constexpr int ACC_OFF = ZERO_OFF + ZERO_BYTES;
  static constexpr int BIAS_OFF = ACC_OFF + 128 * FW_ACC_LD * 4;   // 64 floats
  static constexpr int BAR_OFF = BIAS_OFF + 256;
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;
};
static_assert(FW_A_BYTES % 1024 == 0 && FwSmem::ZERO_OFF % 1024 == 0, "patches and the zero block must stay 1024-aligned");

// M row r of a forward tile holds window position p = r & 3 of pooled pixel fw_pooled(r).  Each group of 8 rows (one
// ldmatrix matrix) pairs two pooled pixels 7 apart, i.e. one pooled row apart: 28 staged pixels, so the group's eight conv
// pixels (+0, +1, +14, +15 and +28, +29, +42, +43) are distinct mod 8 and the gather has no bank conflicts.  Pixels 0-27
// pair as (l, l + 7) within each half; 28-31 pair as (28, 30), (29, 31), conflict-free unless a pooled row ends between.
DMNIST_DEVICE int fw_pooled(int r) {
  const int g = r >> 3, slot = (r >> 2) & 1;
  return g < 14 ? 14 * (g / 7) + 7 * slot + g % 7 : 28 + 2 * slot + (g - 14);
}
DMNIST_DEVICE int fw_row(int l, int p) {
  const int g = l < 28 ? 7 * (l / 14) + l % 7 : 14 + (l & 1);
  const int slot = l < 28 ? (l % 14) / 7 : (l >> 1) & 1;
  return 8 * g + 4 * slot + p;
}

// The pool epilogue stages the 128 x 64 accumulator tile in shared memory; thread = (pooled pixel, 8 channels) then
// reads the four window positions of its channels and stores 16 B of activations and 8 B of pooling codes.
__global__ void __launch_bounds__(CV_THREADS, 1)
conv2_fwd_kernel(const __grid_constant__ CUtensorMap tmX,   // a1 as [B*14 rows][14][32], box (32,14,16,1), 64B swizzle
                 const __grid_constant__ CUtensorMap tmW,   // W [800][64], box (64,200), 128B swizzle
                 const float* __restrict__ bias,            // [64]
                 __nv_bfloat16* __restrict__ out,           // pooled [B,7,7,64]
                 uint8_t* __restrict__ code,                // [B,7,7,64]
                 int num_tiles, int pooled) {               // pooled = B * 49
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + FwSmem::BAR_OFF);
  uint64_t* a_empty = a_full + FW_STAGES;
  uint64_t* w_full = a_empty + FW_STAGES;
  float* s_bias = reinterpret_cast<float*>(smem + FwSmem::BIAS_OFF);
  float* s_acc = reinterpret_cast<float*>(smem + FwSmem::ACC_OFF);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    for (int s = 0; s < FW_STAGES; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], CV_CONSUMERS / 32); }
    mbar_init(w_full, 1);
    fence_mbar_init();
  }
  if (threadIdx.x < 64) s_bias[threadIdx.x] = __ldg(bias + threadIdx.x);
  if (threadIdx.x < ZERO_BYTES / 16) reinterpret_cast<uint4*>(smem + FwSmem::ZERO_OFF)[threadIdx.x] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  pdl_wait();
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(w_full, W_BYTES);
      for (int i = 0; i < 4; ++i) tma_load_2d(smem + i * 25600, &tmW, w_full, 0, 200 * i);
      int it = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++it) {
        // tile = pooled pixels [32t, 32t + 32); its receptive field lies in the 16 stack rows from row0 (rows past the
        // batch are OOB zero fill, and rows the tile does not reach are staged but never read)
        const int q0 = t * FW_POOLED;
        const int row0 = first_staged_row((q0 / 49) * 14 + 2 * ((q0 % 49) / 7));
        const int s = it % FW_STAGES;
        mbar_wait(&a_empty[s], ((it / FW_STAGES) & 1) ^ 1);
        mbar_expect_tx(&a_full[s], FW_A_BYTES);
        tma_load_4d(smem + FwSmem::A_OFF + s * FW_A_BYTES, &tmX, &a_full[s], 0, 0, row0, 0);
      }
    }
    return;
  }

  // ldmatrix rows of this lane: tile row r (tiles 0/1 of x4: rows +0 / +8, tiles 2/3: channel chunk + 1)
  const int r = 16 * warp + (lane & 7) + ((lane >> 3) & 1) * 8;
  const int lr = fw_pooled(r), pr = r & 3, kc = lane >> 4;
  const uint32_t zero = smem_u32(smem + FwSmem::ZERO_OFF);
  // W (MN-major, 128B swizzle): k-row = tap * 32 + ci (128 B = 64 co), 8-row groups 1024 B apart; a tap is 4096 B,
  // a K step of 16 ci 2048 B
  const uint64_t db0 = make_smem_desc(smem_u32(smem), 8192, 1024, SWZ_128B);
  mbar_wait(w_full, 0);
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  int it = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++it) {
    const int q0 = t * FW_POOLED;
    const int row0 = first_staged_row((q0 / 49) * 14 + 2 * ((q0 % 49) / 7));
    // this lane's conv pixel (h, w) of image img; rows of pooled pixels past the batch recompute the last one and are
    // never stored
    const int q = min(q0 + lr, pooled - 1);
    const int img = q / 49, ph = (q % 49) / 7, pw = q % 7;
    const int h = 2 * ph + (pr >> 1), w = 2 * pw + (pr & 1);
    const int pix = (img * 14 + h - row0) * 14 + w;
    const uint32_t inside = inside_taps<1>(h, w);
    const int s = it % FW_STAGES;
    mbar_wait(&a_full[s], (it / FW_STAGES) & 1);
    const uint32_t patch = smem_u32(smem + FwSmem::A_OFF + s * FW_A_BYTES);
    // A fragments (two 16-channel K steps) of one tap; output pixel (h, w) reads pixel (h + kh - 2, w + kw - 2)
    auto load_tap = [&](int tap, uint32_t (&a)[2][4]) {
      const int p = pix + (tap / 5 - 2) * 14 + tap % 5 - 2;
      ldsm_x4(tap_addr<64>(patch, zero, inside, tap, p, kc), a[0]);
      ldsm_x4(tap_addr<64>(patch, zero, inside, tap, p, 2 + kc), a[1]);
    };
    // Two-deep register ring, one commit group per tap: tap + 1 is gathered while tap's wgmmas run.  A buffer is
    // overwritten only after the wgmmas that read it (tap - 1's group) have completed; every wgmma must be able to
    // keep its A registers until its own group retires, or ptxas serializes the whole loop.
    uint32_t a[2][2][4];
    fence_regs(acc);
    load_tap(0, a[0]);
#pragma unroll
    for (int tap = 0; tap < 25; ++tap) {
      wgmma_fence();
      wgmma_m64n64_rs<1>(acc, a[tap & 1][0], desc_advance(db0, tap * 4096), tap != 0);
      wgmma_m64n64_rs<1>(acc, a[tap & 1][1], desc_advance(db0, tap * 4096 + 2048), 1);
      wgmma_commit();
      if (tap + 1 < 25) {
        wgmma_wait<1>();
        load_tap(tap + 1, a[(tap + 1) & 1]);
      }
    }
    wgmma_wait<0>();
    fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&a_empty[s]);

    named_bar_sync(1, CV_CONSUMERS);               // the previous tile's epilogue has read the staging tile
    {
      const int r0 = 16 * warp + (lane >> 2);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        *reinterpret_cast<float2*>(s_acc + r0 * FW_ACC_LD + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(s_acc + (r0 + 8) * FW_ACC_LD + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    named_bar_sync(1, CV_CONSUMERS);
    {
      // 32 pooled pixels x 8 groups of 8 channels
      const int l = threadIdx.x >> 3, cg = threadIdx.x & 7;
      if (q0 + l < pooled) {
        float val[4][8];
#pragma unroll
        for (int p = 0; p < 4; ++p) {                // window position p = dy * 2 + dx
          const float* src = s_acc + fw_row(l, p) * FW_ACC_LD + cg * 8;
          const float4 lo = *reinterpret_cast<const float4*>(src), hi = *reinterpret_cast<const float4*>(src + 4);
          val[p][0] = lo.x; val[p][1] = lo.y; val[p][2] = lo.z; val[p][3] = lo.w;
          val[p][4] = hi.x; val[p][5] = hi.y; val[p][6] = hi.z; val[p][7] = hi.w;
        }
        uint32_t pk[4];
        uint32_t cd[2] = {0u, 0u};
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          float m = val[0][jj];
          uint32_t idx = 0;
#pragma unroll
          for (int p = 1; p < 4; ++p)
            if (val[p][jj] > m) { m = val[p][jj]; idx = p; }
          m += s_bias[cg * 8 + jj];
          const bool active = m > 0.f;
          cd[jj >> 2] |= (idx | (active ? 4u : 0u)) << ((jj & 3) * 8);
          const float o = active ? m : 0.f;
          if (jj & 1) pk[jj >> 1] = pack_bf16x2(__uint_as_float(pk[jj >> 1]), o);
          else pk[jj >> 1] = __float_as_uint(o);
        }
        const size_t off = (size_t)(q0 + l) * 64 + cg * 8;
        *reinterpret_cast<uint4*>(out + off) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
        *reinterpret_cast<uint2*>(code + off) = make_uint2(cd[0], cd[1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------
// dgrad
// ------------------------------------------------------------------------------------------------------
constexpr int DG_ROWS = 14;                    // staged image rows per tile, the most any tile start needs
constexpr int DG_STAGES = 3;
constexpr int DG_A_BYTES = DG_ROWS * 14 * 64 * 2;   // 24.5 KB: 14 rows x 14 pixels x 64 ch
constexpr int DG_A_SLOT = 25 * 1024;                // keeps every patch 1024-aligned (128B swizzle)
static_assert(DG_A_BYTES <= DG_A_SLOT, "a patch runs into the next stage");
struct DgSmem {
  static constexpr int A_OFF = W_BYTES;
  static constexpr int ZERO_OFF = A_OFF + DG_STAGES * DG_A_SLOT;
  static constexpr int BAR_OFF = ZERO_OFF + ZERO_BYTES;
  static constexpr int TOTAL = BAR_OFF + 512 + 1024;
};

__global__ void __launch_bounds__(CV_THREADS, 1)
conv2_dgrad_kernel(const __grid_constant__ CUtensorMap tmDY,  // dY as [B*14 rows][14][64], box (64,14,14,1), 128B swizzle
                   const __grid_constant__ CUtensorMap tmW,
                   __nv_bfloat16* __restrict__ dx,            // [B,14,14,32]
                   int num_tiles, int pixels,                 // pixels = B * 196
                   unsigned long long* __restrict__ dbg) {    // dbg: optional timeline of CTA 0
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + DgSmem::BAR_OFF);
  uint64_t* a_empty = a_full + DG_STAGES;
  uint64_t* w_full = a_empty + DG_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmDY);
    tma_prefetch_desc(&tmW);
    for (int s = 0; s < DG_STAGES; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], CV_CONSUMERS / 32); }
    mbar_init(w_full, 1);
    fence_mbar_init();
  }
  if (threadIdx.x < ZERO_BYTES / 16) reinterpret_cast<uint4*>(smem + DgSmem::ZERO_OFF)[threadIdx.x] = make_uint4(0, 0, 0, 0);
  const bool dbg_on = dbg != nullptr && blockIdx.x == 0;
  if (dbg_on && threadIdx.x == 0) dbg[0] = globaltimer_ns();
  __syncthreads();
  pdl_wait();
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)
  if (dbg_on && threadIdx.x == 0) dbg[1] = globaltimer_ns();

  if (warp == 8) {
    if (lane == 0) {
      mbar_expect_tx(w_full, W_BYTES);
      for (int i = 0; i < 4; ++i) tma_load_2d(smem + i * 25600, &tmW, w_full, 0, 200 * i);
      int it = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++it) {
        const int s = it % DG_STAGES;
        mbar_wait(&a_empty[s], ((it / DG_STAGES) & 1) ^ 1);
        if (dbg_on && it < 20) dbg[8 + it] = globaltimer_ns();          // producer: slot free, issuing load `it`
        mbar_expect_tx(&a_full[s], DG_A_BYTES);
        // tile = pixels [128t, 128t + 128); dX[y,x] += dY[y + 2 - kh, x + 2 - kw] * W[kh,kw] reaches two rows either side
        tma_load_4d(smem + DgSmem::A_OFF + s * DG_A_SLOT, &tmDY, &a_full[s], 0, 0, first_staged_row(t * 128 / 14), 0);
      }
    }
  } else {
    const int r = 16 * warp + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int kc = lane >> 4;
    const uint32_t zero = smem_u32(smem + DgSmem::ZERO_OFF);
    // W[tap] as B: 32 ci rows x 64 co, K-major (128 B rows, 8-row groups 1024 B apart); a K step of 16 co = 32 B
    const uint64_t db0 = make_smem_desc(smem_u32(smem), 16, 1024, SWZ_128B);
    mbar_wait(w_full, 0);
    if (dbg_on && threadIdx.x == 0) dbg[2] = globaltimer_ns();                       // weights resident
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
    int it = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++it) {
      const int g0 = t * 128;
      // this lane's pixel: M row r of the tile; rows past the batch recompute the last pixel and are never stored
      const int g = min(g0 + r, pixels - 1);
      const int row = g / 14, w = g % 14;
      const int pix = g - first_staged_row(g0 / 14) * 14;
      const uint32_t inside = inside_taps<-1>(row % 14, w);
      const int s = it % DG_STAGES;
      mbar_wait(&a_full[s], (it / DG_STAGES) & 1);
      if (dbg_on && threadIdx.x == 0 && it < 20) dbg[32 + it] = globaltimer_ns();   // MMA: data of load `it` landed
      const uint32_t patch = smem_u32(smem + DgSmem::A_OFF + s * DG_A_SLOT);
      // A fragments (four 16-channel K steps) of one tap; tap (kh, kw) reads pixel (h + 2 - kh, w + 2 - kw)
      auto load_tap = [&](int tap, uint32_t (&a)[4][4]) {
        const int p = pix + (2 - tap / 5) * 14 + 2 - tap % 5;
#pragma unroll
        for (int k = 0; k < 4; ++k) ldsm_x4(tap_addr<128>(patch, zero, inside, tap, p, 2 * k + kc), a[k]);
      };
      // Same two-deep register ring as the forward tap loop.
      uint32_t a[2][4][4];
      fence_regs(acc);
      load_tap(0, a[0]);
#pragma unroll
      for (int tap = 0; tap < 25; ++tap) {
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_m64n32_rs<0>(acc, a[tap & 1][k], desc_advance(db0, tap * 4096 + 32 * k), (tap | k) != 0);
        wgmma_commit();
        if (tap + 1 < 25) {
          wgmma_wait<1>();
          load_tap(tap + 1, a[(tap + 1) & 1]);
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&a_empty[s]);
      if (dbg_on && threadIdx.x == 0 && it < 8) dbg[56 + it] = globaltimer_ns();    // accumulator of tile `it` complete
      const int r0 = 16 * warp + (lane >> 2);
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int gg = g0 + r0 + 8 * half;
        if (gg < pixels) {
          __nv_bfloat16* o = dx + (size_t)gg * 32 + 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < 4; ++j)
            *reinterpret_cast<uint32_t*>(o + 8 * j) = pack_bf16x2(acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
        }
      }
    }
  }
  __syncthreads();
  if (dbg_on && threadIdx.x == 0) dbg[3] = globaltimer_ns();
}

// ------------------------------------------------------------------------------------------------------
// wgrad: CTA = (group of 4 taps, slice of the images).  K = the 196 pixels of one image, padded to 208 = 13 K steps of
// 16.  Per image a stage holds the image's 18 x 18 zero-padded input patch (20 KB, A operand for every tap of the
// group) and the image's dY, 208 pixels x 64 co (26 KB, B operand; pixels 196-207 are TMA out-of-bounds zero fill).
// M = (tap, ci): the four taps of a group are 32-row M-chunks (warps 2q, 2q + 1 hold chunk q) whose windows start at
//     group g < 5 : taps (kh = 0..3, kw = g)
//     group 5     : taps (kh = 4, kw = 0..3)
//     group 6     : tap  (kh = 4, kw = 4) + three padding chunks (zero operands, never stored)
// ------------------------------------------------------------------------------------------------------
constexpr int WG_STAGES = 3;
constexpr int WG_KSTEPS = 13;                        // 208 / 16
constexpr int WG_A_BYTES = 18 * 18 * 32 * 2;         // 20736: the patch
constexpr int WG_A_SLOT = 21 * 1024;                 // keeps the dY tile 1024-aligned (128B swizzle)
constexpr int WG_B_BYTES = 16 * WG_KSTEPS * 64 * 2;  // 26624: the dY tile
constexpr int WG_STAGE_BYTES = WG_A_SLOT + WG_B_BYTES;
constexpr int WG_GROUPS = 7;
constexpr int WG_FOLD = 64;                          // images per wgmma accumulator stretch (even: a loop step is 2 images)
static_assert(WG_FOLD % 2 == 0, "the image loop folds at the start of a step");
static_assert(WG_A_BYTES <= WG_A_SLOT, "the patch runs into the dY tile");
struct WgSmem {
  static constexpr int BAR_OFF = WG_STAGES * WG_STAGE_BYTES;
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;   // 145664: a 65 KB conv1_wgrad CTA fits beside it
};
// Partial sums of one tap group of one CTA ([4 M-chunks][32 ci][64 co]), added up in image-slice order by
// conv2_wgrad_reduce_kernel.
constexpr int WG_PART_FLOATS = 4 * 32 * 64;
constexpr int WG_MAX_PARTS = 160;
// One launch of this kernel pair in flight per device: the workspace is static.
__device__ float g_c2wg_part[WG_MAX_PARTS * WG_PART_FLOATS];

// CTA = (tap group, image slice): blockIdx.x = split * WG_GROUPS + group.  Every CTA stores its partial sums: the reduction
// reads all WG_GROUPS * splits slots of the launch.
__global__ void __launch_bounds__(CV_THREADS, 1)
conv2_wgrad_kernel(const __grid_constant__ CUtensorMap tmX,    // a1, box (32,18,18,1), 64B swizzle
                   const __grid_constant__ CUtensorMap tmDY,   // dY as [B][196][64], box (64,208,1), 128B swizzle
                   int B, int splits) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + WgSmem::BAR_OFF);
  uint64_t* empty = full + WG_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int group = blockIdx.x % WG_GROUPS, split = blockIdx.x / WG_GROUPS;
  const int img0 = (int)(((long long)B * split) / splits);
  const int ni = (int)(((long long)B * (split + 1)) / splits) - img0;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmDY);
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], CV_CONSUMERS / 32); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  // (no early launch_dependents: resident-but-blocked CTAs of the next kernel steal SM resources from this one)

  if (warp == 8) {
    if (lane == 0) {
      for (int i = 0; i < ni; ++i) {
        const int s = i % WG_STAGES;
        mbar_wait(&empty[s], ((i / WG_STAGES) & 1) ^ 1);
        uint8_t* st = smem + s * WG_STAGE_BYTES;
        mbar_expect_tx(&full[s], WG_A_BYTES + WG_B_BYTES);
        tma_load_4d(st, &tmX, &full[s], 0, -2, -2, img0 + i);
        tma_load_4d(st + WG_A_SLOT, &tmDY, &full[s], 0, 0, img0 + i, 0);
      }
    }
    return;
  }

  // A^T via ldmatrix.trans: x4 tile i covers ci + 8 (i & 1) and pixels + 8 (i >> 1), so in K step ks this lane supplies
  // the row of pixel p = 16 ks + px, which tap (kh, kw) reads at patch pixel (p / 14 + kh) * 18 + p % 14 + kw.  The pad
  // pixels 196-207 (K step 12, px >= 4) meet zero dY rows; they read patch pixel 0, halo for every tap, so even their
  // products are exact zeros.
  const int q = warp >> 1;                         // M-chunk (tap of the group) of this warp's 16 rows
  const int chunk = 2 * (warp & 1) + ((lane >> 3) & 1);   // 16-byte channel chunk (8 ci)
  const int px = 8 * (lane >> 4) + (lane & 7);
  // patch pixel of this chunk's tap window for image pixel 0; group 6 chunks 1-3 are padding
  const int tap_px = group < 5 ? q * 18 + group : (group == 5 ? 4 * 18 + q : 4 * 18 + 4);
  const bool real_chunk = group < 6 || q == 0;
  // The wgmma accumulator holds at most WG_FOLD images: the tensor cores do not round their fp32 accumulation to nearest,
  // and the error of one accumulator grows with the K steps it collects (a single split of 4133 images came to a
  // normwise 9.1e-4 of the float64 gradient on an H100).  Each full stretch is then added to `folded` in fp32.
  float acc[32], folded[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = folded[j] = 0.f;
  fence_regs(acc);
  // One commit group per K step and a two-deep register ring running across image boundaries, as in the forward tap
  // loop: step k + 1's A fragment is gathered while step k's wgmma runs, and only the wait_group 1 after step k + 1
  // frees step k's registers.  An image's stage is released once the first wgmma of the next image has been issued and
  // the wait after it has returned, i.e. the last wgmma reading the stage has completed.  The loop body covers two images
  // so that the ring's register index is a compile-time constant (13 steps per image).
  uint32_t a[2][4];
  uint32_t patch = 0;
  uint64_t db0 = 0;
  int s = 0, s_prev = 0;
  uint32_t phase = 0;
  for (int i0 = 0; i0 < ni; i0 += 2) {
    if (i0 != 0 && i0 % WG_FOLD == 0) {
      wgmma_wait<0>();
      fence_regs(acc);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        folded[j] += acc[j];
        acc[j] = 0.f;
      }
      fence_regs(acc);
    }
#pragma unroll
    for (int k = 0; k < 2 * WG_KSTEPS; ++k) {
      const int ks = k % WG_KSTEPS;
      if (ks == 0) {
        if (k != 0 && i0 + 1 >= ni) break;
        mbar_wait(&full[s], phase);
        patch = smem_u32(smem + s * WG_STAGE_BYTES);
        // B (MN-major, 128B swizzle): [pixel][64 co], 8-pixel groups 1024 B apart; K step = 16 pixels = 2048 B.
        db0 = make_smem_desc(patch + WG_A_SLOT, 8192, 1024, SWZ_128B);
      }
      if (real_chunk) {
        const int p = 16 * ks + px;
        const int pix = (ks == WG_KSTEPS - 1 && px >= 4) ? 0 : tap_px + p + 4 * (p / 14);
        ldsm_x4_trans(patch_addr<64>(patch, pix, chunk), a[k & 1]);
      } else {
        a[k & 1][0] = a[k & 1][1] = a[k & 1][2] = a[k & 1][3] = 0u;
      }
      wgmma_fence();
      wgmma_m64n64_rs<1>(acc, a[k & 1], desc_advance(db0, 2048 * ks), 1);
      wgmma_commit();
      wgmma_wait<1>();
      if (ks == 0) {
        if (i0 + k > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[s_prev]);
        }
        s_prev = s;
        if (++s == WG_STAGES) { s = 0; phase ^= 1; }
      }
    }
  }
  wgmma_wait<0>();
  fence_regs(acc);
  if (ni > WG_FOLD) {                              // a split of at most WG_FOLD images stores its accumulator as it is
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] += folded[j];
  }

  const int ci0 = 16 * (warp & 1) + (lane >> 2);
  float* part = g_c2wg_part + (size_t)blockIdx.x * WG_PART_FLOATS;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    float* o = part + (q * 32 + ci0 + 8 * half) * 64 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j) *reinterpret_cast<float2*>(o + 8 * j) = make_float2(acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
  }
}

// g_w += the sum of the partials over the image slices, in slice order.  Thread = 4 output channels of one (tap, ci):
// 25 x 32 x 16 = 12800 threads, so the 4 MB of partials are read by the whole machine at once.  Chained to
// conv2_wgrad_kernel by programmatic dependent launch: its launch overlaps the weight-gradient kernel's last CTAs.
// With bias_part, 16 more CTAs add the conv2 bias gradient: g_bias += the sum of dm_fc1_dgrad_unpool_slots' n_bias
// slots in slot order, CTA q channels 4q .. 4q + 3.  In the training step that sum then sits on this side branch, not
// at the end of the data-gradient GEMM.
constexpr int WGR_THREADS = 64;
constexpr int WGR_ITEMS = 25 * 32 * 64 / 4;
constexpr int WGR_CTAS = WGR_ITEMS / WGR_THREADS;
constexpr int WGR_BIAS_CTAS = 16;
static_assert(WGR_ITEMS % WGR_THREADS == 0, "every thread of the weight CTAs owns an item");
__global__ void __launch_bounds__(WGR_THREADS)
conv2_wgrad_reduce_kernel(float* __restrict__ g_w, int splits, const float* __restrict__ bias_part, int n_bias,
                          float* __restrict__ g_bias) {
  __shared__ float4 s_buf[4 * WGR_THREADS];
  pdl_wait();
  if (blockIdx.x >= WGR_CTAS) {
    add_ordered_slot_sum64<WGR_THREADS>(bias_part, n_bias, blockIdx.x - WGR_CTAS, g_bias, s_buf);
    return;
  }
  const int e4 = blockIdx.x * WGR_THREADS + threadIdx.x;
  const int tap = e4 >> 9, row4 = e4 & 511;        // row4 = ci * 16 + co / 4
  const int kh = tap / 5, kw = tap % 5;
  const int group = kh < 4 ? kw : (kw < 4 ? 5 : 6);
  const int q = kh < 4 ? kh : (kw < 4 ? kw : 0);
  const float4 sum = ordered_sum4(reinterpret_cast<const float4*>(g_c2wg_part + (size_t)group * WG_PART_FLOATS) + q * 512 + row4,
                                  splits, (size_t)WG_GROUPS * WG_PART_FLOATS / 4);
  float4* o = reinterpret_cast<float4*>(g_w) + e4;
  const float4 cur = *o;
  *o = make_float4(cur.x + sum.x, cur.y + sum.y, cur.z + sum.z, cur.w + sum.w);
}

int launch_conv2_wgrad(const void* a1, const void* dy, void* g_w, const void* bias_part, int n_bias, void* g_bias,
                       int B, void* stream) {
  CUtensorMap tmX, tmDY;
  if (make_tmap_nhwc_bf16(&tmX, a1, 32, 14, 14, B, 32, 18, 18, 64)) return 101;
  // dY viewed as [B][196 pixels][64 co]: the 208-pixel box ends in zero fill rather than in the next image
  if (make_tmap_nhwc_bf16(&tmDY, dy, 64, 196, B, 1, 64, 16 * WG_KSTEPS, 1, 128)) return 102;
  int splits = max_ctas() / WG_GROUPS;
  if (splits * WG_GROUPS > WG_MAX_PARTS) splits = WG_MAX_PARTS / WG_GROUPS;
  if (splits > B) splits = B;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(conv2_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WgSmem::TOTAL));
    DM_CUDA_OK(cudaFuncSetAttribute(conv2_wgrad_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DM_CUDA_OK(launch_kernel(conv2_wgrad_kernel, dim3(WG_GROUPS * splits), dim3(CV_THREADS), WgSmem::TOTAL, st, tmX, tmDY,
                           B, splits));
  return (int)launch_kernel(conv2_wgrad_reduce_kernel, dim3(WGR_CTAS + (bias_part ? WGR_BIAS_CTAS : 0)), dim3(WGR_THREADS),
                            0, st, reinterpret_cast<float*>(g_w), splits, reinterpret_cast<const float*>(bias_part),
                            n_bias, reinterpret_cast<float*>(g_bias));
}

}  // namespace dm

extern "C" {

// a1: [B,14,14,32] bf16;  w_bf16: HWIO [800][64] bf16;  out/code: [B,7,7,64]
int dm_conv2_fwd(const void* a1, const void* w_bf16, const void* bias, void* out, void* code, int B, void* stream) {
  using namespace dm;
  CUtensorMap tmX, tmW;
  if (make_tmap_nhwc_bf16(&tmX, a1, 32, 14, 14 * B, 1, 32, 14, FW_ROWS, 64)) return 101;
  if (make_tmap_2d_bf16(&tmW, w_bf16, 64, 800, 64, 64, 200, 128)) return 102;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(conv2_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FwSmem::TOTAL));
    DM_CUDA_OK(cudaFuncSetAttribute(conv2_fwd_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  const int tiles = (B * 49 + FW_POOLED - 1) / FW_POOLED;
  const int grid = tiles < num_sms() ? tiles : num_sms();
  return (int)launch_kernel(conv2_fwd_kernel, dim3(grid), dim3(CV_THREADS), FwSmem::TOTAL,
                            reinterpret_cast<cudaStream_t>(stream), tmX, tmW, reinterpret_cast<const float*>(bias),
                            reinterpret_cast<__nv_bfloat16*>(out), reinterpret_cast<uint8_t*>(code), tiles, B * 49);
}

// dy: [B,14,14,64] bf16 -> dx: [B,14,14,32] bf16
int dm_conv2_dgrad(const void* dy, const void* w_bf16, void* dx, int B, void* stream) {
  using namespace dm;
  CUtensorMap tmDY, tmW;
  if (make_tmap_nhwc_bf16(&tmDY, dy, 64, 14, 14 * B, 1, 64, 14, DG_ROWS, 128)) return 101;
  if (make_tmap_2d_bf16(&tmW, w_bf16, 64, 800, 64, 64, 200, 128)) return 102;
  static bool configured = false;
  if (!configured) {
    DM_CUDA_OK(cudaFuncSetAttribute(conv2_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, DgSmem::TOTAL));
    DM_CUDA_OK(cudaFuncSetAttribute(conv2_dgrad_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    configured = true;
  }
  const int tiles = (B * 196 + 127) / 128;
  const int grid = tiles < max_ctas() ? tiles : max_ctas();
  return (int)launch_kernel(conv2_dgrad_kernel, dim3(grid), dim3(CV_THREADS), DgSmem::TOTAL,
                            reinterpret_cast<cudaStream_t>(stream), tmDY, tmW, reinterpret_cast<__nv_bfloat16*>(dx), tiles,
                            B * 196, static_cast<unsigned long long*>(nullptr));
}

// g_w ([25][32][64] fp32) must be zeroed by the caller; the gradient is added to it.  Two launches: the weight-gradient
// kernel and the reduction of its partial sums.
int dm_conv2_wgrad(const void* a1, const void* dy, void* g_w, int B, void* stream) {
  return dm::launch_conv2_wgrad(a1, dy, g_w, nullptr, 0, nullptr, B, stream);
}

// The same, and g_bias ([64] fp32, pre-zeroed) += the sum of the n_bias conv2 bias-gradient slots that
// dm_fc1_dgrad_unpool_slots stored into bias_part, in slot order: what dm_fc1_dgrad_unpool adds, to the bit.
int dm_conv2_wgrad_bias(const void* a1, const void* dy, void* g_w, const void* bias_part, int n_bias, void* g_bias, int B,
                        void* stream) {
  if (bias_part == nullptr || g_bias == nullptr || n_bias < 1) return -1;
  return dm::launch_conv2_wgrad(a1, dy, g_w, bias_part, n_bias, g_bias, B, stream);
}

}  // extern "C"
