// ktb_runtime.cu — device registry, peer access, arenas, CUDA IPC, error strings.
//
// Replaces, on the local-GPU route, the rendezvous/membership half of the reference:
// kt/serving/distributed_supervisor.py:90-174 (pod_ips quorum) becomes a static table of
// local devices with NVLink peer access enabled between every pair.
#include "ktb_common.cuh"

#include <stdarg.h>
#include <atomic>
#include <mutex>
#include <unordered_map>

namespace ktb {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

const char* last_error_cstr() { return g_err; }
void host_workers_shutdown();   // ktb_host.cu
void host_blocks_shutdown();    // ktb_host.cu

static std::mutex g_mu;
static DeviceInfo g_dev[kMaxDevices];
static std::atomic<bool> g_registered[kMaxDevices];   // publication flag: set after g_dev[d] is fully built
static bool g_peer[kMaxDevices][kMaxDevices];
struct HostBlock { size_t nbytes; };
static std::unordered_map<void*, size_t> g_arena[kMaxDevices];
static std::unordered_map<void*, size_t> g_host;
static std::unordered_map<void*, int> g_ipc_open;

DeviceInfo* device_info(int dev) {
  if (dev < 0 || dev >= kMaxDevices) return nullptr;
  return g_registered[dev].load(std::memory_order_acquire) ? &g_dev[dev] : nullptr;
}

int require_device(int dev) {
  if (!device_info(dev)) {
    set_error("device %d is not registered: call ktb_init first", dev);
    return KTB_ERR_STATE;
  }
  return KTB_OK;
}

static int register_device(int dev) {
  DeviceInfo& d = g_dev[dev];
  if (d.registered) return KTB_OK;
  KTB_GUARD(dev);
  cudaDeviceProp prop;
  KTB_CK(cudaGetDeviceProperties(&prop, dev));
  KTB_REQUIRE(prop.major == 9 && prop.minor == 0, KTB_ERR_UNSUPPORTED,
              "device %d is sm_%d%d; libktb200 carries sm_90a code only", dev, prop.major, prop.minor);
  d.sm_count = prop.multiProcessorCount;
  KTB_CK(cudaStreamCreateWithFlags(&d.stream_h2d, cudaStreamNonBlocking));
  KTB_CK(cudaStreamCreateWithFlags(&d.stream_exec, cudaStreamNonBlocking));
  KTB_CK(cudaStreamCreateWithFlags(&d.stream_d2h, cudaStreamNonBlocking));
  KTB_CK(cudaStreamCreateWithFlags(&d.stream_rank, cudaStreamNonBlocking));
  KTB_CK(cudaStreamCreateWithFlags(&d.stream_stage, cudaStreamNonBlocking));
  for (int i = 0; i < 6; ++i) KTB_CK(cudaEventCreateWithFlags(&d.host_ev[i], cudaEventDisableTiming));
  d.registered = true;
  g_peer[dev][dev] = true;
  g_registered[dev].store(true, std::memory_order_release);
  return KTB_OK;
}

static int enable_peer(int dev, int peer) {
  if (g_peer[dev][peer]) return KTB_OK;
  int can = 0;
  KTB_CK(cudaDeviceCanAccessPeer(&can, dev, peer));
  if (!can) return KTB_OK;  // stays false; callers check ktb_peer_enabled
  KTB_GUARD(dev);
  cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();  // clear sticky-less error
  } else if (e != cudaSuccess) {
    set_error("cudaDeviceEnablePeerAccess(%d->%d) failed: %s", dev, peer, cudaGetErrorString(e));
    return KTB_ERR_CUDA;
  }
  g_peer[dev][peer] = true;
  return KTB_OK;
}

}  // namespace ktb

using namespace ktb;

extern "C" {

int ktb_version(void) { return KTB_VERSION; }

const char* ktb_last_error(void) { return g_err; }

int ktb_init(int n_dev, const int* dev_ids) {
  KTB_REQUIRE(n_dev > 0 && dev_ids, KTB_ERR_ARG, "ktb_init: need at least one device id");
  int count = 0;
  KTB_CK(cudaGetDeviceCount(&count));
  std::lock_guard<std::mutex> lk(g_mu);
  for (int i = 0; i < n_dev; ++i) {
    int d = dev_ids[i];
    KTB_REQUIRE(d >= 0 && d < count && d < kMaxDevices, KTB_ERR_ARG,
                "ktb_init: device id %d out of range (visible devices: %d)", d, count);
    int rc = register_device(d);
    if (rc) return rc;
  }
  // NVSwitch gives every pair full bandwidth: enable every ordered pair among registered devices.
  for (int a = 0; a < kMaxDevices; ++a)
    for (int b = 0; b < kMaxDevices; ++b)
      if (a != b && g_dev[a].registered && g_dev[b].registered) {
        int rc = enable_peer(a, b);
        if (rc) return rc;
      }
  return KTB_OK;
}

int ktb_shutdown(void) {
  host_workers_shutdown();
  host_blocks_shutdown();
  std::lock_guard<std::mutex> lk(g_mu);
  for (auto& kv : g_ipc_open) {   // peers' arenas mapped into this process
    if (kv.second >= 0 && kv.second < kMaxDevices && g_dev[kv.second].registered) {
      DeviceGuard g(kv.second);
      cudaIpcCloseMemHandle(kv.first);
    }
  }
  g_ipc_open.clear();
  for (int d = 0; d < kMaxDevices; ++d) {
    if (!g_dev[d].registered) continue;
    g_registered[d].store(false, std::memory_order_release);
    DeviceGuard g(d);
    cudaDeviceSynchronize();
    for (auto& kv : g_arena[d]) cudaFree(kv.first);
    g_arena[d].clear();
    cudaStreamDestroy(g_dev[d].stream_h2d);
    cudaStreamDestroy(g_dev[d].stream_exec);
    cudaStreamDestroy(g_dev[d].stream_d2h);
    cudaStreamDestroy(g_dev[d].stream_rank);
    cudaStreamDestroy(g_dev[d].stream_stage);
    for (int i = 0; i < 6; ++i) cudaEventDestroy(g_dev[d].host_ev[i]);
    g_dev[d] = DeviceInfo();
  }
  for (auto& kv : g_host) cudaFreeHost(kv.first);
  g_host.clear();
  for (int a = 0; a < kMaxDevices; ++a)
    for (int b = 0; b < kMaxDevices; ++b) g_peer[a][b] = false;
  return KTB_OK;
}

int ktb_sm_count(int dev) {
  int rc = require_device(dev);
  if (rc) return rc;
  return device_info(dev)->sm_count;
}

int ktb_peer_enabled(int dev, int peer) {
  if (dev < 0 || dev >= kMaxDevices || peer < 0 || peer >= kMaxDevices) {
    set_error("ktb_peer_enabled: bad device ids %d,%d", dev, peer);
    return KTB_ERR_ARG;
  }
  return g_peer[dev][peer] ? 1 : 0;
}

int ktb_arena_alloc(int dev, size_t nbytes, void** out) {
  KTB_REQUIRE(out && nbytes > 0, KTB_ERR_ARG, "ktb_arena_alloc: null out or zero size");
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_GUARD(dev);
  void* p = nullptr;
  KTB_CK(cudaMalloc(&p, nbytes));
  std::lock_guard<std::mutex> lk(g_mu);
  g_arena[dev][p] = nbytes;
  *out = p;
  return KTB_OK;
}

int ktb_arena_free(int dev, void* ptr) {
  int rc = require_device(dev);
  if (rc) return rc;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_arena[dev].find(ptr);
    KTB_REQUIRE(it != g_arena[dev].end(), KTB_ERR_ARG,
                "ktb_arena_free: %p is not an arena of device %d", ptr, dev);
    g_arena[dev].erase(it);
  }
  KTB_GUARD(dev);
  KTB_CK(cudaFree(ptr));
  return KTB_OK;
}

int ktb_host_alloc(size_t nbytes, void** out) {
  KTB_REQUIRE(out && nbytes > 0, KTB_ERR_ARG, "ktb_host_alloc: null out or zero size");
  void* p = nullptr;
  KTB_CK(cudaHostAlloc(&p, nbytes, cudaHostAllocPortable | cudaHostAllocMapped));
  std::lock_guard<std::mutex> lk(g_mu);
  g_host[p] = nbytes;
  *out = p;
  return KTB_OK;
}

int ktb_host_free(void* ptr) {
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_host.find(ptr);
    KTB_REQUIRE(it != g_host.end(), KTB_ERR_ARG, "ktb_host_free: %p was not allocated here", ptr);
    g_host.erase(it);
  }
  KTB_CK(cudaFreeHost(ptr));
  return KTB_OK;
}

int ktb_ipc_export(int dev, void* ptr, unsigned char handle[KTB_IPC_HANDLE_BYTES]) {
  static_assert(sizeof(cudaIpcMemHandle_t) == KTB_IPC_HANDLE_BYTES, "IPC handle size");
  KTB_REQUIRE(ptr && handle, KTB_ERR_ARG, "ktb_ipc_export: null argument");
  int rc = require_device(dev);
  if (rc) return rc;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    KTB_REQUIRE(g_arena[dev].count(ptr), KTB_ERR_ARG,
                "ktb_ipc_export: %p is not the base of a ktb_arena_alloc block on device %d", ptr, dev);
  }
  KTB_GUARD(dev);
  cudaIpcMemHandle_t h;
  KTB_CK(cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle, &h, sizeof(h));
  return KTB_OK;
}

int ktb_ipc_open(int dev, const unsigned char handle[KTB_IPC_HANDLE_BYTES], void** out) {
  KTB_REQUIRE(handle && out, KTB_ERR_ARG, "ktb_ipc_open: null argument");
  int rc = require_device(dev);
  if (rc) return rc;
  KTB_GUARD(dev);
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void* p = nullptr;
  KTB_CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  std::lock_guard<std::mutex> lk(g_mu);
  g_ipc_open[p] = dev;
  *out = p;
  return KTB_OK;
}

int ktb_ipc_close(int dev, void* ptr) {
  int rc = require_device(dev);
  if (rc) return rc;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_ipc_open.find(ptr);
    KTB_REQUIRE(it != g_ipc_open.end(), KTB_ERR_ARG, "ktb_ipc_close: %p was not opened here", ptr);
    g_ipc_open.erase(it);
  }
  KTB_GUARD(dev);
  KTB_CK(cudaIpcCloseMemHandle(ptr));
  return KTB_OK;
}

int ktb_shard_bounds(size_t n, int world, int rank, size_t* begin, size_t* end) {
  KTB_REQUIRE(world > 0 && rank >= 0 && rank < world && begin && end, KTB_ERR_ARG,
              "ktb_shard_bounds: bad world/rank %d/%d", world, rank);
  size_t chunk = (n + (size_t)world - 1) / (size_t)world;  // torch.chunk: ceil(n / world)
  size_t b = chunk * (size_t)rank;
  if (b > n) b = n;
  size_t e = b + chunk;
  if (e > n) e = n;
  *begin = b;
  *end = e;
  return KTB_OK;
}

}  // extern "C"
