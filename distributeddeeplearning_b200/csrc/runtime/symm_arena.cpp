// Symmetric (peer-mapped) device arena with optional NVLS multicast alias.
//
// This is the native replacement for the transport setup the reference inherits from
// NCCL/MPI (SURVEY.md 2.4, N3): every rank allocates the same-sized physical arena with the
// CUDA VMM API, exports it as a POSIX fd, imports the 7 peers' arenas and maps them into its
// own address space.  Kernels then address `peer_ptrs[r] + offset` directly over NVLink.
// When the fabric supports it, one multicast object is bound over all arenas; stores to /
// reductions from `mc_ptr + offset` are replicated / reduced inside the NVSwitch
// (multimem.st / multimem.ld_reduce).
//
// libcuda is opened lazily with dlopen so this module imports on a GPU-less build box.
#include "host_runtime.h"

#include <cuda.h>
#include <dlfcn.h>
#include <unistd.h>

#include <cstring>
#include <mutex>
#include <stdexcept>

namespace ddl {
namespace {

struct Driver {
  void* lib = nullptr;
  bool ok = false;
  CUresult (*Init)(unsigned int) = nullptr;
  CUresult (*GetErrorString)(CUresult, const char**) = nullptr;
  CUresult (*DeviceGet)(CUdevice*, int) = nullptr;
  CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  CUresult (*DevicePrimaryCtxRetain)(CUcontext*, CUdevice) = nullptr;
  CUresult (*CtxSetCurrent)(CUcontext) = nullptr;
  CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*,
                                          CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*,
                        unsigned long long) = nullptr;
  CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle,
                                         CUmemAllocationHandleType, unsigned long long) = nullptr;
  CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*,
                                           CUmemAllocationHandleType) = nullptr;
  CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle,
                     unsigned long long) = nullptr;
  CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*MemsetD8)(CUdeviceptr, unsigned char, size_t) = nullptr;
  CUresult (*CtxSynchronize)() = nullptr;
  CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle,
                               size_t, size_t, unsigned long long) = nullptr;
  CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*,
                                      CUmulticastGranularity_flags) = nullptr;
};

Driver& drv() {
  static Driver d;
  static std::once_flag once;
  std::call_once(once, []() {
    d.lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!d.lib) return;
    bool all = true;
    auto sym = [&](const char* name, bool required = true) -> void* {
      void* p = dlsym(d.lib, name);
      if (!p && required) all = false;
      return p;
    };
#define DDL_LOAD(field, name) d.field = reinterpret_cast<decltype(d.field)>(sym(name))
#define DDL_LOAD_OPT(field, name) d.field = reinterpret_cast<decltype(d.field)>(sym(name, false))
    DDL_LOAD(Init, "cuInit");
    DDL_LOAD(GetErrorString, "cuGetErrorString");
    DDL_LOAD(DeviceGet, "cuDeviceGet");
    DDL_LOAD(DeviceGetAttribute, "cuDeviceGetAttribute");
    DDL_LOAD(DevicePrimaryCtxRetain, "cuDevicePrimaryCtxRetain");
    DDL_LOAD(CtxSetCurrent, "cuCtxSetCurrent");
    DDL_LOAD(MemGetAllocationGranularity, "cuMemGetAllocationGranularity");
    DDL_LOAD(MemCreate, "cuMemCreate");
    DDL_LOAD(MemRelease, "cuMemRelease");
    DDL_LOAD(MemExportToShareableHandle, "cuMemExportToShareableHandle");
    DDL_LOAD(MemImportFromShareableHandle, "cuMemImportFromShareableHandle");
    DDL_LOAD(MemAddressReserve, "cuMemAddressReserve");
    DDL_LOAD(MemAddressFree, "cuMemAddressFree");
    DDL_LOAD(MemMap, "cuMemMap");
    DDL_LOAD(MemUnmap, "cuMemUnmap");
    DDL_LOAD(MemSetAccess, "cuMemSetAccess");
    DDL_LOAD(MemsetD8, "cuMemsetD8_v2");
    DDL_LOAD(CtxSynchronize, "cuCtxSynchronize");
    DDL_LOAD_OPT(MulticastCreate, "cuMulticastCreate");
    DDL_LOAD_OPT(MulticastAddDevice, "cuMulticastAddDevice");
    DDL_LOAD_OPT(MulticastBindMem, "cuMulticastBindMem");
    DDL_LOAD_OPT(MulticastGetGranularity, "cuMulticastGetGranularity");
#undef DDL_LOAD
#undef DDL_LOAD_OPT
    d.ok = all;
  });
  return d;
}

std::string cu_err(CUresult r) {
  const char* s = nullptr;
  if (drv().GetErrorString && drv().GetErrorString(r, &s) == CUDA_SUCCESS && s) return s;
  return "CUresult " + std::to_string(static_cast<int>(r));
}

#define DDL_CU(call)                                                                      \
  do {                                                                                    \
    CUresult _r = (call);                                                                 \
    if (_r != CUDA_SUCCESS) throw std::runtime_error(std::string(#call) + ": " + cu_err(_r)); \
  } while (0)

size_t round_up(size_t x, size_t m) { return (x + m - 1) / m * m; }

CUmemAllocationProp alloc_prop(int device) {
  CUmemAllocationProp prop;
  std::memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  return prop;
}

CUmulticastObjectProp mc_prop(int world, size_t bytes) {
  CUmulticastObjectProp p;
  std::memset(&p, 0, sizeof(p));
  p.numDevices = static_cast<unsigned int>(world);
  p.size = bytes;
  p.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  p.flags = 0;
  return p;
}

uint64_t map_handle(CUmemGenericAllocationHandle h, size_t bytes, size_t gran, int device) {
  CUdeviceptr va = 0;
  DDL_CU(drv().MemAddressReserve(&va, bytes, gran, 0, 0));
  try {
    DDL_CU(drv().MemMap(va, bytes, 0, h, 0));
    CUmemAccessDesc acc;
    std::memset(&acc, 0, sizeof(acc));
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    DDL_CU(drv().MemSetAccess(va, bytes, &acc, 1));
  } catch (...) {
    drv().MemAddressFree(va, bytes);
    throw;
  }
  return static_cast<uint64_t>(va);
}

}  // namespace

bool driver_available() { return drv().ok; }

SymmArena::SymmArena(int rank, int world, int device, size_t bytes)
    : rank_(rank), world_(world), device_(device), req_bytes_(bytes) {
  if (rank < 0 || world < 1 || rank >= world) throw std::invalid_argument("SymmArena: bad rank/world");
  if (bytes == 0) throw std::invalid_argument("SymmArena: zero bytes");
}

SymmArena::~SymmArena() { release(); }

bool SymmArena::multicast_supported() const {
  if (!drv().ok || !drv().MulticastCreate) return false;
  CUdevice dev;
  if (drv().DeviceGet(&dev, device_) != CUDA_SUCCESS) return false;
  int v = 0;
  if (drv().DeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) != CUDA_SUCCESS) return false;
  return v != 0;
}

void SymmArena::alloc() {
  if (!drv().ok) throw std::runtime_error("SymmArena: libcuda.so.1 not available");
  DDL_CU(drv().Init(0));
  CUdevice dev;
  DDL_CU(drv().DeviceGet(&dev, device_));
  CUcontext ctx;
  DDL_CU(drv().DevicePrimaryCtxRetain(&ctx, dev));
  DDL_CU(drv().CtxSetCurrent(ctx));
  CUmemAllocationProp prop = alloc_prop(device_);
  size_t gran = 0;
  DDL_CU(drv().MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
  if (world_ > 1 && multicast_supported() && drv().MulticastGetGranularity) {
    CUmulticastObjectProp mp = mc_prop(world_, round_up(req_bytes_, gran));
    size_t mgran = 0;
    if (drv().MulticastGetGranularity(&mgran, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS &&
        mgran > gran)
      gran = mgran;
  }
  gran_ = gran;
  bytes_ = round_up(req_bytes_, gran_);
  CUmemGenericAllocationHandle h;
  DDL_CU(drv().MemCreate(&h, bytes_, &prop, 0));
  handle_ = h;
  ptrs_.assign(world_, 0);
  peer_handles_.assign(world_, 0);
  ptrs_[rank_] = map_handle(h, bytes_, gran_, device_);
  DDL_CU(drv().MemsetD8(static_cast<CUdeviceptr>(ptrs_[rank_]), 0, bytes_));
  DDL_CU(drv().CtxSynchronize());
}

void SymmArena::exchange(const std::string& session, int timeout_ms) {
  if (world_ <= 1) return;
  if (!handle_) throw std::runtime_error("SymmArena::exchange before alloc");
  int fd = -1;
  DDL_CU(drv().MemExportToShareableHandle(&fd, handle_, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  std::vector<int> fds;
  try {
    fds = exchange_fds(rank_, world_, fd, session, timeout_ms);
  } catch (...) {
    ::close(fd);
    throw;
  }
  ::close(fd);
  std::string err;
  for (int r = 0; r < world_; ++r) {
    if (r == rank_) continue;
    if (err.empty()) {
      try {
        CUmemGenericAllocationHandle h;
        DDL_CU(drv().MemImportFromShareableHandle(&h, reinterpret_cast<void*>(static_cast<uintptr_t>(fds[r])),
                                                  CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
        peer_handles_[r] = h;
        ptrs_[r] = map_handle(h, bytes_, gran_, device_);
      } catch (const std::exception& e) {
        err = e.what();
      }
    }
    if (fds[r] >= 0) ::close(fds[r]);
  }
  if (!err.empty()) throw std::runtime_error("SymmArena::exchange: " + err);
}

bool SymmArena::mc_create(const std::string& session, int timeout_ms) {
  if (world_ <= 1 || !multicast_supported()) return false;
  try {
    CUdevice dev;
    DDL_CU(drv().DeviceGet(&dev, device_));
    CUmulticastObjectProp mp = mc_prop(world_, bytes_);
    int fd = -1;
    CUmemGenericAllocationHandle mc = 0;
    if (rank_ == 0) {
      DDL_CU(drv().MulticastCreate(&mc, &mp));
      DDL_CU(drv().MemExportToShareableHandle(&fd, mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    }
    int got = broadcast_fd(rank_, world_, 0, fd, session, timeout_ms);
    if (rank_ != 0) {
      DDL_CU(drv().MemImportFromShareableHandle(&mc, reinterpret_cast<void*>(static_cast<uintptr_t>(got)),
                                                CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
    }
    if (got >= 0) ::close(got);
    mc_handle_ = mc;
    DDL_CU(drv().MulticastAddDevice(mc, dev));
    mc_added_ = true;
    return true;
  } catch (const std::exception& e) {
    err_ = e.what();
    return false;
  }
}

bool SymmArena::mc_bind() {
  if (!mc_added_) return false;
  try {
    DDL_CU(drv().MulticastBindMem(mc_handle_, 0, handle_, 0, bytes_, 0));
    mc_ptr_ = map_handle(mc_handle_, bytes_, gran_, device_);
    return true;
  } catch (const std::exception& e) {
    err_ = e.what();
    mc_ptr_ = 0;
    return false;
  }
}

void SymmArena::release() {
  if (!drv().ok) return;
  if (mc_ptr_) {
    drv().MemUnmap(static_cast<CUdeviceptr>(mc_ptr_), bytes_);
    drv().MemAddressFree(static_cast<CUdeviceptr>(mc_ptr_), bytes_);
    mc_ptr_ = 0;
  }
  if (mc_handle_) {
    drv().MemRelease(mc_handle_);
    mc_handle_ = 0;
  }
  for (size_t r = 0; r < ptrs_.size(); ++r) {
    if (ptrs_[r]) {
      drv().MemUnmap(static_cast<CUdeviceptr>(ptrs_[r]), bytes_);
      drv().MemAddressFree(static_cast<CUdeviceptr>(ptrs_[r]), bytes_);
      ptrs_[r] = 0;
    }
    if (r < peer_handles_.size() && peer_handles_[r]) {
      drv().MemRelease(peer_handles_[r]);
      peer_handles_[r] = 0;
    }
  }
  if (handle_) {
    drv().MemRelease(handle_);
    handle_ = 0;
  }
}

}  // namespace ddl
