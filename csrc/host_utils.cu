#include "host_utils.h"

#include <mutex>

namespace dm {

int g_pdl = 0;
int g_max_ctas = 0;

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess &&
        v > 0)
      n = v;
    else
      return 1;
  }
  return n;
}

void* driver_symbol(const char* name) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess) {
    fprintf(stderr, "[dmnist] driver symbol %s unavailable (err %d, query %d)\n", name, (int)e, (int)qres);
    (void)cudaGetLastError();
    return nullptr;
  }
  return fn;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] { fn = reinterpret_cast<EncodeTiledFn>(driver_symbol("cuTensorMapEncodeTiled")); });
  return fn;
}

static CUtensorMapSwizzle swizzle_enum(int bytes) {
  switch (bytes) {
    case 32: return CU_TENSOR_MAP_SWIZZLE_32B;
    case 64: return CU_TENSOR_MAP_SWIZZLE_64B;
    case 128: return CU_TENSOR_MAP_SWIZZLE_128B;
    default: return CU_TENSOR_MAP_SWIZZLE_NONE;
  }
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t ld_elems,
                      uint32_t box_inner, uint32_t box_outer, int swizzle_bytes) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return 1;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld_elems * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_enum(swizzle_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[dmnist] cuTensorMapEncodeTiled(2d) failed: %d (base=%p inner=%llu outer=%llu ld=%llu box=%u,%u)\n",
            (int)r, base, (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld_elems,
            box_inner, box_outer);
    return 2;
  }
  return 0;
}

int make_tmap_nhwc_bf16(CUtensorMap* out, const void* base, int C, int W, int H, int N, uint32_t box_c,
                        uint32_t box_w, uint32_t box_h, int swizzle_bytes) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return 1;
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {box_c, box_w, box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_enum(swizzle_bytes), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[dmnist] cuTensorMapEncodeTiled(4d) failed: %d (C=%d W=%d H=%d N=%d box=%u,%u,%u)\n", (int)r, C,
            W, H, N, box_c, box_w, box_h);
    return 2;
  }
  return 0;
}

}  // namespace dm

extern "C" int dm_version() { return 2; }

// n outside [8, SM count] (0 included) restores the default: one CTA per SM.
extern "C" int dm_set_max_ctas(int n) {
  dm::g_max_ctas = (n >= 8 && n <= dm::num_sms()) ? n : 0;
  return dm::max_ctas();
}

// The grid bound set by dm_set_max_ctas, 0 when the default is in force (so callers can put it back).
extern "C" int dm_get_max_ctas() { return dm::g_max_ctas; }

extern "C" int dm_num_sms() { return dm::num_sms(); }

// The largest batch every kernel of the LeNet training step and evaluation accepts (DESIGN.md §3, "Batch limit"):
// fc1_dgrad_unpool's 4096 bias-gradient slots at 49 per 128-row tile (10 624 rows) and fc2_fwd_bwd's 65 536 per-row
// loss slots.  Every other LeNet kernel loops over the batch or caps its grid, and the evaluation runs in chunks of
// at most dm_eval_max_rows() rows whatever the batch.
extern "C" int dm_lenet_max_batch() {
  const int a = dm::fc1_dgrad_unpool_max_batch(), b = dm::fc2_fwd_bwd_max_batch();
  return a < b ? a : b;
}

extern "C" int dm_set_pdl(int on) {
  dm::g_pdl = on ? 1 : 0;
  return dm::g_pdl;
}

// Device query used by the Python side to fail loudly on parts other than sm_90.
extern "C" int dm_device_cc(int device) {
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return -1;
  return prop.major * 10 + prop.minor;
}
