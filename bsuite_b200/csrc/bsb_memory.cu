// Compressible device memory for observation buffers (bsb_obs_malloc / bsb_obs_free / bsb_obs_memory_info).
//
// Observations are mostly zero: a deep_sea tile is 4 KB holding at most one 1.0f, a catch board 50 cells with two
// ones, an mnist LAST frame nothing at all.  Memory created with cuMemCreate(compressionType =
// CU_MEM_ALLOCATION_COMP_GENERIC) is compressed by the L2 on its way to DRAM, so writing such tiles moves far fewer
// DRAM bytes; kernels and copy engines still see ordinary memory, and the values read back are the values written.
//
// The driver calls are resolved through cudaGetDriverEntryPoint, so the library keeps linking cudart statically and
// nothing else.  Every request is served: when the device cannot compress, the compressible backing store is used up
// (it is finite) or the driver hands back an allocation without compression, the request falls back to cudaMalloc.
// The two kinds are counted separately per device (bsb_obs_memory_info).
#include <cuda.h>

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>

#include "bsb_env.h"

namespace bsb {
namespace {

struct Driver {
  decltype(&cuDeviceGetAttribute) get_attribute = nullptr;
  decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
  decltype(&cuMemCreate) create = nullptr;
  decltype(&cuMemGetAllocationPropertiesFromHandle) properties = nullptr;
  decltype(&cuMemAddressReserve) reserve = nullptr;
  decltype(&cuMemMap) map = nullptr;
  decltype(&cuMemSetAccess) set_access = nullptr;
  decltype(&cuMemUnmap) unmap = nullptr;
  decltype(&cuMemRelease) release = nullptr;
  decltype(&cuMemAddressFree) address_free = nullptr;
  bool ok = false;
};

template <typename F>
bool resolve(const char* name, F* fn) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult found = cudaDriverEntryPointSymbolNotFound;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &found) != cudaSuccess ||
      found != cudaDriverEntryPointSuccess || p == nullptr)
    return false;
  *fn = reinterpret_cast<F>(p);
  return true;
}

const Driver& driver() {
  static Driver d;
  static std::once_flag once;
  std::call_once(once, [] {
    d.ok = resolve("cuDeviceGetAttribute", &d.get_attribute) &&
           resolve("cuMemGetAllocationGranularity", &d.granularity) && resolve("cuMemCreate", &d.create) &&
           resolve("cuMemGetAllocationPropertiesFromHandle", &d.properties) &&
           resolve("cuMemAddressReserve", &d.reserve) && resolve("cuMemMap", &d.map) &&
           resolve("cuMemSetAccess", &d.set_access) && resolve("cuMemUnmap", &d.unmap) &&
           resolve("cuMemRelease", &d.release) && resolve("cuMemAddressFree", &d.address_free);
  });
  return d;
}

struct Block {
  int device;
  size_t bytes;                          // reserved and mapped (compressed) or requested (plain)
  CUmemGenericAllocationHandle handle;   // compressed blocks only
  bool compressed;
};

struct Counters { uint64_t compressed = 0, plain = 0; };

std::mutex g_mutex;
std::map<uintptr_t, Block> g_blocks;               // every live pointer bsb_obs_malloc returned, by address
std::unordered_map<int, Counters> g_counters;      // per device ordinal
std::atomic<int64_t> g_live_compressed{0};         // compressed blocks in g_blocks (launches skip the lookup at 0)

struct DeviceGuard {
  int prev = 0; bool ok;
  explicit DeviceGuard(int dev) { ok = cudaGetDevice(&prev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess; }
  ~DeviceGuard() { if (ok) cudaSetDevice(prev); }
};

// BSB_OK when `device` names a CUDA device of this process
int check_device(int device) {
  if (device < 0) return fail(BSB_INVALID_ARGUMENT, "bsb_obs_malloc: device must be a CUDA ordinal (host buffers are plain host memory)");
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(BSB_CUDA_ERROR, std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e));
  }
  if (device >= count)
    return fail(BSB_INVALID_ARGUMENT, "device " + std::to_string(device) + " does not exist (" + std::to_string(count) + " CUDA devices)");
  return BSB_OK;
}

int compression_supported(const Driver& d, int device) {
  int value = 0;
  if (!d.ok || d.get_attribute(&value, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, device) != CUDA_SUCCESS) return 0;
  return value;
}

// A compressible mapping of at least `size` bytes, or 0 when the driver does not grant one.
CUdeviceptr map_compressed(const Driver& d, int device, size_t size, Block* block) {
  CUmemAllocationProp prop = {};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  prop.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
  size_t granularity = 0;
  if (d.granularity(&granularity, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS || granularity == 0) return 0;
  const size_t bytes = (size + granularity - 1) / granularity * granularity;
  CUmemGenericAllocationHandle handle;
  if (d.create(&handle, bytes, &prop, 0) != CUDA_SUCCESS) return 0;   // e.g. the compressible backing store is used up
  CUmemAllocationProp granted = {};
  if (d.properties(&granted, handle) != CUDA_SUCCESS || granted.allocFlags.compressionType != CU_MEM_ALLOCATION_COMP_GENERIC) {
    d.release(handle);
    return 0;
  }
  CUdeviceptr ptr = 0;
  if (d.reserve(&ptr, bytes, granularity, 0, 0) != CUDA_SUCCESS) {
    d.release(handle);
    return 0;
  }
  CUmemAccessDesc access = {};
  access.location = prop.location;
  access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if (d.map(ptr, bytes, 0, handle, 0) != CUDA_SUCCESS) {
    d.address_free(ptr, bytes);
    d.release(handle);
    return 0;
  }
  if (d.set_access(ptr, bytes, &access, 1) != CUDA_SUCCESS) {
    d.unmap(ptr, bytes);
    d.address_free(ptr, bytes);
    d.release(handle);
    return 0;
  }
  *block = Block{device, bytes, handle, true};
  return ptr;
}

}  // namespace

bool in_compressed_block(const void* p) {
  if (g_live_compressed.load(std::memory_order_relaxed) == 0) return false;
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  std::lock_guard<std::mutex> lock(g_mutex);
  auto it = g_blocks.upper_bound(a);
  if (it == g_blocks.begin()) return false;
  --it;
  return it->second.compressed && a - it->first < it->second.bytes;
}

}  // namespace bsb

extern "C" {

void* bsb_obs_malloc(ptrdiff_t size, int device, void* stream) {
  (void)stream;   // creation and mapping are not stream-ordered
  using namespace bsb;
  if (size < 0) { fail(BSB_INVALID_ARGUMENT, "bsb_obs_malloc: size must be >= 0"); return nullptr; }
  if (check_device(device) != BSB_OK) return nullptr;
  if (size == 0) return nullptr;
  DeviceGuard guard(device);
  if (!guard.ok) { cudaGetLastError(); fail(BSB_CUDA_ERROR, "bsb_obs_malloc: cudaSetDevice failed"); return nullptr; }
  const Driver& d = driver();
  Block block{};
  void* ptr = nullptr;
  if (compression_supported(d, device))
    ptr = reinterpret_cast<void*>(map_compressed(d, device, static_cast<size_t>(size), &block));
  if (ptr == nullptr) {
    cudaError_t e = cudaMalloc(&ptr, static_cast<size_t>(size));
    if (e != cudaSuccess) {
      cudaGetLastError();
      fail(e == cudaErrorMemoryAllocation ? BSB_OUT_OF_MEMORY : BSB_CUDA_ERROR,
           std::string("bsb_obs_malloc: cudaMalloc: ") + cudaGetErrorString(e));
      return nullptr;
    }
    block = Block{device, static_cast<size_t>(size), 0, false};
  }
  std::lock_guard<std::mutex> lock(g_mutex);
  g_blocks[reinterpret_cast<uintptr_t>(ptr)] = block;
  Counters& c = g_counters[device];
  (block.compressed ? c.compressed : c.plain) += block.bytes;
  if (block.compressed) g_live_compressed.fetch_add(1, std::memory_order_relaxed);
  return ptr;
}

void bsb_obs_free(void* ptr, ptrdiff_t size, int device, void* stream) {
  (void)size; (void)device; (void)stream;   // the table knows the block
  using namespace bsb;
  if (ptr == nullptr) return;
  Block block;
  {
    std::lock_guard<std::mutex> lock(g_mutex);
    auto it = g_blocks.find(reinterpret_cast<uintptr_t>(ptr));
    if (it == g_blocks.end()) { fail(BSB_INVALID_ARGUMENT, "bsb_obs_free: pointer was not returned by bsb_obs_malloc"); return; }
    block = it->second;
    g_blocks.erase(it);
    Counters& c = g_counters[block.device];
    (block.compressed ? c.compressed : c.plain) -= block.bytes;
    if (block.compressed) g_live_compressed.fetch_sub(1, std::memory_order_relaxed);
  }
  DeviceGuard guard(block.device);
  if (block.compressed) {
    // cudaFree waits for the device before it releases memory, and torch's caching allocator relies on that when it
    // hands segments back; cuMemUnmap does not wait, so wait here.
    cudaDeviceSynchronize();
    const Driver& d = driver();
    const CUdeviceptr p = reinterpret_cast<CUdeviceptr>(ptr);
    d.unmap(p, block.bytes);
    d.address_free(p, block.bytes);
    d.release(block.handle);
  } else {
    cudaFree(ptr);
  }
}

int32_t bsb_obs_memory_info(int device, int32_t* supported, uint64_t* compressed_bytes, uint64_t* plain_bytes) {
  using namespace bsb;
  if (supported == nullptr || compressed_bytes == nullptr || plain_bytes == nullptr)
    return fail(BSB_INVALID_ARGUMENT, "bsb_obs_memory_info: null output pointer");
  if (int status = check_device(device)) return status;
  *supported = compression_supported(driver(), device);
  std::lock_guard<std::mutex> lock(g_mutex);
  const Counters c = g_counters[device];
  *compressed_bytes = c.compressed;
  *plain_bytes = c.plain;
  return BSB_OK;
}

}  // extern "C"
