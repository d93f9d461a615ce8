// Symmetric memory: every rank allocates the same buffers and maps every peer's copy, so
// kernels address peer memory directly over NVLink (the transport that replaces the
// reference's gRPC parameter-server traffic, SURVEY §5.8).
//
// Backend 1 (always available): cudaMalloc + CUDA IPC handles.  The 64-byte handles are exchanged
// by the Python side over the existing process group; opening a handle enables peer access lazily.
//
// Backend 2 (NVSwitch systems): CUDA virtual memory management + an **NVLS multicast object**, set up here with
// the driver API (no dependence on torch's private symmetric-memory module):
//     every rank   cuMemCreate (POSIX-fd shareable, device-pinned)  -> export fd -> peers import + map it (P2P view)
//     rank 0       cuMulticastCreate(numDevices = N)                 -> export fd -> peers import
//     every rank   cuMulticastAddDevice; <barrier>; cuMulticastBindMem(own physical handle); <barrier>;
//                  reserve VA + cuMemMap(multicast handle) -> the address whose loads are reduced inside the switch
//                  (multimem.ld_reduce) and whose stores are replicated to every rank (multimem.st).
// File descriptors travel between the processes over AF_UNIX sockets (SCM_RIGHTS), done by the Python side
// (parallel/symm_mem.py); the barriers are process-group barriers.
#include <string.h>
#include <unistd.h>

#include <mutex>
#include <vector>

#include "host_utils.h"

namespace dm {

#define DM_DRV_OK(expr)                                                                                     \
  do {                                                                                                      \
    CUresult _r = (expr);                                                                                   \
    if (_r != CUDA_SUCCESS) {                                                                               \
      fprintf(stderr, "[dmnist] driver error %d at %s:%d: %s\n", (int)_r, __FILE__, __LINE__, #expr);       \
      return 1000 + (int)_r;                                                                                \
    }                                                                                                       \
  } while (0)

struct VmmApi {
  CUresult (*DeviceGet)(CUdevice*, int);
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice);
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags);
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long);
  CUresult (*MemRelease)(CUmemGenericAllocationHandle);
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long);
  CUresult (*MemAddressFree)(CUdeviceptr, size_t);
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
  CUresult (*MemUnmap)(CUdeviceptr, size_t);
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t);
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long);
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType);
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*);
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice);
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long);
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags);
  bool ok = false;
};

static VmmApi* vmm_api() {
  static VmmApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    bool ok = true;
#define DM_SYM(field, name)                                              \
  api.field = reinterpret_cast<decltype(api.field)>(driver_symbol(name)); \
  ok = ok && api.field != nullptr
    DM_SYM(DeviceGet, "cuDeviceGet");
    DM_SYM(DeviceGetAttribute, "cuDeviceGetAttribute");
    DM_SYM(MemGetAllocationGranularity, "cuMemGetAllocationGranularity");
    DM_SYM(MemCreate, "cuMemCreate");
    DM_SYM(MemRelease, "cuMemRelease");
    DM_SYM(MemAddressReserve, "cuMemAddressReserve");
    DM_SYM(MemAddressFree, "cuMemAddressFree");
    DM_SYM(MemMap, "cuMemMap");
    DM_SYM(MemUnmap, "cuMemUnmap");
    DM_SYM(MemSetAccess, "cuMemSetAccess");
    DM_SYM(MemExportToShareableHandle, "cuMemExportToShareableHandle");
    DM_SYM(MemImportFromShareableHandle, "cuMemImportFromShareableHandle");
    DM_SYM(MulticastCreate, "cuMulticastCreate");
    DM_SYM(MulticastAddDevice, "cuMulticastAddDevice");
    DM_SYM(MulticastBindMem, "cuMulticastBindMem");
    DM_SYM(MulticastGetGranularity, "cuMulticastGetGranularity");
#undef DM_SYM
    api.ok = ok;
  });
  return api.ok ? &api : nullptr;
}

static CUmemAllocationProp device_prop(int device) {
  CUmemAllocationProp prop;
  memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return prop;
}

// Reserve a VA range, map `h` into it and grant this device read/write access.
static int map_handle(VmmApi* api, CUmemGenericAllocationHandle h, size_t bytes, size_t align, int device, CUdeviceptr* out) {
  CUdeviceptr va = 0;
  DM_DRV_OK(api->MemAddressReserve(&va, bytes, align, 0, 0));
  CUresult r = api->MemMap(va, bytes, 0, h, 0);
  if (r != CUDA_SUCCESS) {
    api->MemAddressFree(va, bytes);
    fprintf(stderr, "[dmnist] cuMemMap failed: %d\n", (int)r);
    return 1000 + (int)r;
  }
  CUmemAccessDesc acc;
  memset(&acc, 0, sizeof(acc));
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = device;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  r = api->MemSetAccess(va, bytes, &acc, 1);
  if (r != CUDA_SUCCESS) {
    api->MemUnmap(va, bytes);
    api->MemAddressFree(va, bytes);
    fprintf(stderr, "[dmnist] cuMemSetAccess failed: %d\n", (int)r);
    return 1000 + (int)r;
  }
  *out = va;
  return 0;
}

}  // namespace dm

extern "C" {

int dm_set_device(int device) {
  DM_CUDA_OK(cudaSetDevice(device));
  DM_CUDA_OK(cudaFree(0));
  return 0;
}

int dm_symm_alloc(unsigned long long bytes, void** out) {
  void* p = nullptr;
  DM_CUDA_OK(cudaMalloc(&p, bytes));
  DM_CUDA_OK(cudaMemset(p, 0, bytes));
  DM_CUDA_OK(cudaDeviceSynchronize());
  *out = p;
  return 0;
}

int dm_symm_ipc_handle(void* p, void* handle64) {
  cudaIpcMemHandle_t h;
  DM_CUDA_OK(cudaIpcGetMemHandle(&h, p));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &h, sizeof(h));
  return 0;
}

int dm_symm_ipc_open(const void* handle64, void** out) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, sizeof(h));
  void* p = nullptr;
  DM_CUDA_OK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  *out = p;
  return 0;
}

int dm_symm_ipc_close(void* p) {
  DM_CUDA_OK(cudaIpcCloseMemHandle(p));
  return 0;
}

int dm_memset_async(void* p, int value, unsigned long long bytes, void* stream) {
  DM_CUDA_OK(cudaMemsetAsync(p, value, bytes, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}


// ---- backend 2: VMM + NVLS multicast -----------------------------------------------------------------------------------------

// 1 if the device can take part in a multicast object (NVSwitch fabric with NVLS), 0 if not, < 0 on error.
int dm_vmm_multicast_supported(int device) {
  using namespace dm;
  VmmApi* api = vmm_api();
  if (!api) return -1;
  CUdevice dev;
  if (api->DeviceGet(&dev, device) != CUDA_SUCCESS) return -2;
  int v = 0;
  if (api->DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) != CUDA_SUCCESS) return -3;
  return v;
}

// Allocation size every rank must use for a symmetric buffer of `bytes` shared by `ndev` devices: a multiple of both
// the physical-allocation granularity and the multicast granularity.
long long dm_vmm_round_size(unsigned long long bytes, int device, int ndev) {
  using namespace dm;
  VmmApi* api = vmm_api();
  if (!api) return -1;
  CUmemAllocationProp prop = device_prop(device);
  size_t g1 = 0, g2 = 0;
  if (api->MemGetAllocationGranularity(&g1, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS) return -2;
  if (ndev > 1) {
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof(mp));
    mp.numDevices = (unsigned)ndev;
    mp.size = bytes;
    mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    if (api->MulticastGetGranularity(&g2, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) != CUDA_SUCCESS) g2 = 0;
  }
  size_t g = g1 > g2 ? g1 : g2;
  if (g == 0) return -3;
  return (long long)((bytes + g - 1) / g * g);
}

// Physical allocation on `device` (zero-initialised), mapped locally; returns the handle, its POSIX fd and the local address.
int dm_vmm_create(unsigned long long bytes, int device, unsigned long long* handle_out, int* fd_out, void** ptr_out) {
  using namespace dm;
  VmmApi* api = vmm_api();
  if (!api) return -1;
  CUmemAllocationProp prop = device_prop(device);
  CUmemGenericAllocationHandle h;
  DM_DRV_OK(api->MemCreate(&h, bytes, &prop, 0));
  int fd = -1;
  DM_DRV_OK(api->MemExportToShareableHandle(&fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  CUdeviceptr va = 0;
  int rc = map_handle(api, h, bytes, 0, device, &va);
  if (rc) return rc;
  DM_CUDA_OK(cudaMemset(reinterpret_cast<void*>(va), 0, bytes));
  DM_CUDA_OK(cudaDeviceSynchronize());
  *handle_out = (unsigned long long)h;
  *fd_out = fd;
  *ptr_out = reinterpret_cast<void*>(va);
  return 0;
}

// Import a peer's (or the multicast object's) fd; the fd stays owned by the caller.
int dm_vmm_import(int fd, unsigned long long* handle_out) {
  using namespace dm;
  VmmApi* api = vmm_api();
  if (!api) return -1;
  CUmemGenericAllocationHandle h;
  DM_DRV_OK(api->MemImportFromShareableHandle(&h, reinterpret_cast<void*>(static_cast<uintptr_t>(fd)),
                                              CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
  *handle_out = (unsigned long long)h;
  return 0;
}

// Map an (imported) handle into this process for `device`.
int dm_vmm_map(unsigned long long handle, unsigned long long bytes, int device, void** ptr_out) {
  using namespace dm;
  VmmApi* api = vmm_api();
  if (!api) return -1;
  CUdeviceptr va = 0;
  int rc = map_handle(api, (CUmemGenericAllocationHandle)handle, bytes, 0, device, &va);
  if (rc) return rc;
  *ptr_out = reinterpret_cast<void*>(va);
  return 0;
}

int dm_close_fd(int fd) { return close(fd); }

// Rank 0: create the multicast object for `ndev` devices and export its fd.
int dm_mc_create(unsigned long long bytes, int ndev, unsigned long long* handle_out, int* fd_out) {
  using namespace dm;
  VmmApi* api = vmm_api();
  if (!api) return -1;
  CUmulticastObjectProp mp;
  memset(&mp, 0, sizeof(mp));
  mp.numDevices = (unsigned)ndev;
  mp.size = bytes;
  mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  CUmemGenericAllocationHandle mc;
  DM_DRV_OK(api->MulticastCreate(&mc, &mp));
  int fd = -1;
  DM_DRV_OK(api->MemExportToShareableHandle(&fd, mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  *handle_out = (unsigned long long)mc;
  *fd_out = fd;
  return 0;
}

int dm_mc_add_device(unsigned long long mc, int device) {
  using namespace dm;
  VmmApi* api = vmm_api();
  if (!api) return -1;
  CUdevice dev;
  DM_DRV_OK(api->DeviceGet(&dev, device));
  DM_DRV_OK(api->MulticastAddDevice((CUmemGenericAllocationHandle)mc, dev));
  return 0;
}

// After EVERY device has been added: bind this rank's physical allocation at offset 0 of the multicast object.
int dm_mc_bind(unsigned long long mc, unsigned long long mem_handle, unsigned long long bytes) {
  using namespace dm;
  VmmApi* api = vmm_api();
  if (!api) return -1;
  DM_DRV_OK(api->MulticastBindMem((CUmemGenericAllocationHandle)mc, 0, (CUmemGenericAllocationHandle)mem_handle, 0, bytes, 0));
  return 0;
}

}  // extern "C"
