// ktb_host.cu — the host-resident form of the remote-map call: args and results live in pinned HOST memory
// (the reference's client sits outside the GPU: kt/serving/http_client.py:1041-1111 → pod → back), shard r
// moves host → GPU r → host over GPU r's own PCIe link.
//
// What makes this scale past one GPU (round-1 finding: one issuing thread + one buffer on NUMA node 0 capped the
// whole box at ~130-180 GB/s whatever N was):
//   * one persistent ISSUE THREAD per registered GPU, bound to the CPUs of that GPU's NUMA node: every GPU's
//     H2D → kernel → D2H chunk pipeline is enqueued concurrently, and each thread only waits for its own GPU;
//   * NUMA-SHARDED pinned buffers (ktb_host_alloc_sharded): the pages of shard r are first-touched by GPU r's
//     issue thread, i.e. on GPU r's NUMA node, before the block is page-locked (cudaHostRegister), so no DMA
//     crosses the socket interconnect.
// One entry, ktb_map_host_multi, serves every host-path call: one GPU, all ranks, a subset of the ranks (NULL
// staging), and ranks that share a GPU (they run one after another in that GPU's job).
// Replaces, for host-resident tensors, the whole client→pod→client round trip of the reference
// (serving/utils.py:730-749 pack, process_pool.py:125-234 queues, http_server.py:1768-1842 decode/encode,
// serving/utils.py:787-813 unpack).
#include "ktb_common.cuh"

#include <sched.h>
#include <sys/mman.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <vector>

namespace ktb {

// ---- NUMA topology from sysfs (no libnuma in the image) --------------------------------------------------
static int read_int_file(const char* path, int fallback) {
  FILE* f = fopen(path, "r");
  if (!f) return fallback;
  int v = fallback;
  if (fscanf(f, "%d", &v) != 1) v = fallback;
  fclose(f);
  return v;
}

static int device_numa_node_uncached(int dev) {
  char bdf[32] = {0};
  if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), dev) != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  for (char* c = bdf; *c; ++c) *c = (char)tolower(*c);
  char path[128];
  snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bdf);
  return read_int_file(path, -1);
}

// CPUs of a NUMA node ("0-31,64-95") → cpu_set_t; false if unknown.
static bool node_cpuset(int node, cpu_set_t* set) {
  if (node < 0) return false;
  char path[128];
  snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
  FILE* f = fopen(path, "r");
  if (!f) return false;
  char buf[1024] = {0};
  bool ok = fgets(buf, sizeof(buf), f) != nullptr;
  fclose(f);
  if (!ok) return false;
  CPU_ZERO(set);
  int n = 0;
  for (char* tok = strtok(buf, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
    int a = 0, b = 0;
    if (sscanf(tok, "%d-%d", &a, &b) == 2) {
    } else if (sscanf(tok, "%d", &a) == 1) {
      b = a;
    } else {
      continue;
    }
    for (int c = a; c <= b && c < CPU_SETSIZE; ++c) {
      CPU_SET(c, set);
      ++n;
    }
  }
  return n > 0;
}

// ---- per-device issue threads ----------------------------------------------------------------------------
struct HostWorker {
  int dev = -1;
  int numa = -1;
  std::thread th;
  std::mutex mu;
  std::condition_variable cv;
  std::function<int()> job;   // returns a ktb_status; the message is copied into `err`
  bool has_job = false, done = false, stop = false;
  int rc = KTB_OK;
  char err[512] = "";
};

static std::mutex g_workers_mu;
static HostWorker* g_workers[kMaxDevices] = {nullptr};
static std::atomic<int> g_numa_cache[kMaxDevices];
static std::atomic<bool> g_numa_known[kMaxDevices];

static int device_numa_node(int dev) {
  if (dev < 0 || dev >= kMaxDevices) return -1;
  if (!g_numa_known[dev].load()) {
    g_numa_cache[dev] = device_numa_node_uncached(dev);
    g_numa_known[dev] = true;
  }
  return g_numa_cache[dev];
}

const char* last_error_cstr();   // ktb_runtime.cu

static void worker_loop(HostWorker* w) {
  cpu_set_t set;
  if (node_cpuset(w->numa, &set)) {
    cpu_set_t allowed;
    if (sched_getaffinity(0, sizeof(allowed), &allowed) == 0) {
      cpu_set_t both;
      CPU_AND(&both, &set, &allowed);
      if (CPU_COUNT(&both) > 0) sched_setaffinity(0, sizeof(both), &both);
    }
  }
  cudaSetDevice(w->dev);
  std::unique_lock<std::mutex> lk(w->mu);
  for (;;) {
    w->cv.wait(lk, [&] { return w->has_job || w->stop; });
    if (w->stop) return;
    std::function<int()> job = std::move(w->job);
    w->has_job = false;
    lk.unlock();
    int rc = job();
    lk.lock();
    w->rc = rc;
    if (rc != KTB_OK) snprintf(w->err, sizeof(w->err), "%s", last_error_cstr());
    w->done = true;
    w->cv.notify_all();
  }
}

static HostWorker* worker_for(int dev) {
  std::lock_guard<std::mutex> lk(g_workers_mu);
  if (!g_workers[dev]) {
    HostWorker* w = new HostWorker();
    w->dev = dev;
    w->numa = device_numa_node(dev);
    w->th = std::thread(worker_loop, w);
    g_workers[dev] = w;
  }
  return g_workers[dev];
}

static void worker_post(HostWorker* w, std::function<int()> job) {
  std::lock_guard<std::mutex> lk(w->mu);
  w->job = std::move(job);
  w->has_job = true;
  w->done = false;
  w->cv.notify_all();
}

static int worker_wait(HostWorker* w) {
  std::unique_lock<std::mutex> lk(w->mu);
  w->cv.wait(lk, [&] { return w->done; });
  if (w->rc != KTB_OK) set_error("%s", w->err);
  return w->rc;
}

void host_workers_shutdown() {   // called from ktb_shutdown
  std::lock_guard<std::mutex> lk(g_workers_mu);
  for (int d = 0; d < kMaxDevices; ++d) {
    HostWorker* w = g_workers[d];
    if (!w) continue;
    {
      std::lock_guard<std::mutex> l2(w->mu);
      w->stop = true;
      w->cv.notify_all();
    }
    if (w->th.joinable()) w->th.join();
    delete w;
    g_workers[d] = nullptr;
  }
}

// ---- the chunk pipeline of ONE device (runs on whichever thread calls it) ----------------------------------
// H2D copy, kernel and D2H copy of successive chunks overlap on three streams (PCIe is full duplex); staging
// buffers are double-buffered (2 * chunk_bytes each).  Returns after dst_host is complete.
static int run_host_pipeline(int dev, int op, int dtype, const uint8_t* src_host, uint8_t* dst_host, size_t n_bytes,
                             const MapParams& p, size_t chunk_bytes, void* stage_in, void* stage_out) {
  if (n_bytes == 0) return KTB_OK;
  KTB_GUARD(dev);
  DeviceInfo* di = device_info(dev);
  const size_t es = dtype_size(dtype);
  const size_t n_chunks = (n_bytes + chunk_bytes - 1) / chunk_bytes;
  int status = KTB_OK;
  for (size_t c = 0; c < n_chunks && status == KTB_OK; ++c) {
    const int b = (int)(c & 1);
    cudaEvent_t h2d_done = di->host_ev[b], exec_done = di->host_ev[2 + b], d2h_done = di->host_ev[4 + b];
    const size_t off = c * chunk_bytes;
    const size_t len = std::min(chunk_bytes, n_bytes - off);
    uint8_t* sin = static_cast<uint8_t*>(stage_in) + (size_t)b * chunk_bytes;
    uint8_t* sout = static_cast<uint8_t*>(stage_out) + (size_t)b * chunk_bytes;
    cudaError_t e = cudaSuccess;
    if (c >= 2) e = cudaStreamWaitEvent(di->stream_h2d, exec_done, 0);   // stage_in[b] consumed
    if (e == cudaSuccess) e = cudaMemcpyAsync(sin, src_host + off, len, cudaMemcpyHostToDevice, di->stream_h2d);
    if (e == cudaSuccess) e = cudaEventRecord(h2d_done, di->stream_h2d);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(di->stream_exec, h2d_done, 0);
    if (e == cudaSuccess && c >= 2) e = cudaStreamWaitEvent(di->stream_exec, d2h_done, 0);   // stage_out[b] drained
    if (e == cudaSuccess) {
      status = launch_map(dev, op, dtype, sin, sout, len / es, p, KTB_VARIANT_AUTO, di->stream_exec);
      if (status != KTB_OK) break;
      e = cudaEventRecord(exec_done, di->stream_exec);
    }
    if (e == cudaSuccess) e = cudaStreamWaitEvent(di->stream_d2h, exec_done, 0);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dst_host + off, sout, len, cudaMemcpyDeviceToHost, di->stream_d2h);
    if (e == cudaSuccess) e = cudaEventRecord(d2h_done, di->stream_d2h);
    if (e != cudaSuccess) {
      set_error("host pipeline: device %d chunk %zu failed: %s", dev, c, cudaGetErrorString(e));
      status = KTB_ERR_CUDA;
    }
  }
  // the last D2H copy is ordered after every kernel and every H2D copy of this call
  cudaError_t e1 = cudaStreamSynchronize(di->stream_d2h);
  cudaError_t e2 = (status == KTB_OK) ? cudaSuccess : cudaStreamSynchronize(di->stream_exec);
  cudaError_t e3 = (status == KTB_OK) ? cudaSuccess : cudaStreamSynchronize(di->stream_h2d);
  if (status == KTB_OK && (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess)) {
    set_error("host pipeline: stream sync on device %d failed: %s", dev, cudaGetErrorString(e1));
    status = KTB_ERR_CUDA;
  }
  return status;
}

static std::mutex g_host_call_mu;   // the per-device copy/exec streams and events carry one call at a time

struct HostBlockInfo {
  size_t len;       // mmap length
  void* base;       // mmap base (may precede the aligned user pointer)
};
static std::mutex g_sharded_mu;
static std::unordered_map<void*, HostBlockInfo> g_sharded;

void host_blocks_shutdown() {
  std::lock_guard<std::mutex> lk(g_sharded_mu);
  for (auto& kv : g_sharded) {
    cudaHostUnregister(kv.first);
    munmap(kv.second.base, kv.second.len);
  }
  g_sharded.clear();
}

}  // namespace ktb

using namespace ktb;

extern "C" {

int ktb_device_numa_node(int dev) {
  int rc = require_device(dev);
  if (rc) return rc;
  int node = device_numa_node(dev);
  return node < 0 ? -1 : node;
}

int ktb_host_alloc_sharded(size_t nbytes, int n_parts, const size_t* part_end, const int* part_dev, void** out) {
  KTB_REQUIRE(out && nbytes > 0, KTB_ERR_ARG, "ktb_host_alloc_sharded: null out or zero size");
  KTB_REQUIRE(n_parts >= 0 && n_parts <= kMaxDevices && (n_parts == 0 || (part_end && part_dev)), KTB_ERR_ARG,
              "ktb_host_alloc_sharded: bad partition arguments");
  size_t prev = 0;
  for (int i = 0; i < n_parts; ++i) {
    KTB_REQUIRE(part_end[i] >= prev && part_end[i] <= nbytes, KTB_ERR_ARG,
                "ktb_host_alloc_sharded: part_end must be non-decreasing and <= nbytes");
    int rc = require_device(part_dev[i]);
    if (rc) return rc;
    prev = part_end[i];
  }
  // the issue threads carry one job at a time (single-slot mailboxes): allocations and host-path calls take turns
  std::lock_guard<std::mutex> lk(g_host_call_mu);
  constexpr size_t kHuge = 2u << 20;
  const size_t len = (nbytes + kHuge - 1) / kHuge * kHuge + kHuge;
  void* base = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  KTB_REQUIRE(base != MAP_FAILED, KTB_ERR_CUDA, "ktb_host_alloc_sharded: mmap of %zu bytes failed", len);
  uint8_t* p = reinterpret_cast<uint8_t*>(((uintptr_t)base + kHuge - 1) / kHuge * kHuge);
  madvise(p, len - (size_t)(p - static_cast<uint8_t*>(base)), MADV_HUGEPAGE);   // best effort
  // first touch, part by part, from the issue thread of the part's GPU (= on that GPU's NUMA node)
  const size_t page = (size_t)sysconf(_SC_PAGESIZE);
  std::vector<HostWorker*> posted;
  size_t b = 0;
  for (int i = 0; i < n_parts; ++i) {
    // boundaries rounded to pages so every page has exactly one toucher
    size_t e = (i == n_parts - 1) ? nbytes : std::min(nbytes, (part_end[i] + page / 2) / page * page);
    if (e > b) {
      HostWorker* w = worker_for(part_dev[i]);
      // a worker takes one job at a time: wait for an earlier part on the same device first
      if (std::find(posted.begin(), posted.end(), w) != posted.end()) {
        worker_wait(w);
        posted.erase(std::find(posted.begin(), posted.end(), w));
      }
      uint8_t* lo = p + b;
      const size_t n = e - b;
      worker_post(w, [lo, n]() {
        memset(lo, 0, n);
        return (int)KTB_OK;
      });
      posted.push_back(w);
    }
    b = std::max(b, e);
  }
  for (HostWorker* w : posted) worker_wait(w);
  if (b < nbytes) memset(p + b, 0, nbytes - b);
  cudaError_t e = cudaHostRegister(p, nbytes, cudaHostRegisterPortable | cudaHostRegisterMapped);
  if (e != cudaSuccess) {
    munmap(base, len);
    set_error("ktb_host_alloc_sharded: cudaHostRegister(%zu bytes) failed: %s", nbytes, cudaGetErrorString(e));
    return KTB_ERR_CUDA;
  }
  {
    std::lock_guard<std::mutex> lk(g_sharded_mu);
    g_sharded[p] = HostBlockInfo{len, base};
  }
  *out = p;
  return KTB_OK;
}

int ktb_host_free_sharded(void* ptr) {
  HostBlockInfo info;
  {
    std::lock_guard<std::mutex> lk(g_sharded_mu);
    auto it = g_sharded.find(ptr);
    KTB_REQUIRE(it != g_sharded.end(), KTB_ERR_ARG, "ktb_host_free_sharded: %p was not allocated here", ptr);
    info = it->second;
    g_sharded.erase(it);
  }
  KTB_CK(cudaHostUnregister(ptr));
  munmap(info.base, info.len);
  return KTB_OK;
}

int ktb_map_host_multi(int op, int dtype, const void* src_host, void* dst_host, size_t n_elems, size_t granule,
                       double alpha, double beta, int n_ranks, const int* devs, size_t chunk_bytes,
                       void* const* stage_in, void* const* stage_out) {
  int rc = check_dtype("ktb_map_host_multi", dtype);
  if (rc) return rc;
  KTB_REQUIRE(n_ranks > 0 && n_ranks <= kMaxDevices && devs && stage_in && stage_out, KTB_ERR_ARG,
              "ktb_map_host_multi: bad rank arguments");
  if (n_elems == 0) return KTB_OK;
  KTB_REQUIRE(src_host && dst_host, KTB_ERR_ARG, "ktb_map_host_multi: null host buffer");
  KTB_REQUIRE(granule > 0 && n_elems % granule == 0, KTB_ERR_ARG, "ktb_map_host_multi: n_elems not a multiple of granule");
  KTB_REQUIRE(chunk_bytes >= 4096 && chunk_bytes % 256 == 0, KTB_ERR_ARG,
              "ktb_map_host_multi: chunk_bytes must be a multiple of 256 and >= 4096 (got %zu)", chunk_bytes);
  for (int r = 0; r < n_ranks; ++r) {
    rc = require_device(devs[r]);
    if (rc) return rc;
    KTB_REQUIRE((stage_in[r] == nullptr) == (stage_out[r] == nullptr), KTB_ERR_ARG,
                "ktb_map_host_multi: rank %d has one staging buffer (both, or neither to skip the rank)", r);
  }
  rc = check_elementwise("ktb_map_host_multi", op, dtype);   // before any rank's pipeline starts
  if (rc) return rc;
  const size_t es = dtype_size(dtype);
  const size_t rows = n_elems / granule;
  std::lock_guard<std::mutex> lk(g_host_call_mu);
  const MapParams p = make_params(alpha, beta, dtype);
  const uint8_t* src = static_cast<const uint8_t*>(src_host);
  uint8_t* dst = static_cast<uint8_t*>(dst_host);
  // one job per device: its selected ranks in rank order, one after another, since they share the device's
  // streams, events and staging buffers
  auto run_device = [=](int dev) {
    int status = KTB_OK;
    for (int r = 0; r < n_ranks && status == KTB_OK; ++r) {
      if (devs[r] != dev || !stage_in[r]) continue;
      size_t b = 0, e = 0;
      ktb_shard_bounds(rows, n_ranks, r, &b, &e);
      const size_t off = b * granule * es;
      status = run_host_pipeline(dev, op, dtype, src + off, dst + off, (e - b) * granule * es, p, chunk_bytes,
                                 stage_in[r], stage_out[r]);
    }
    return status;
  };
  int jobs[kMaxDevices];   // devices with at least one selected, non-empty rank, in order of first appearance
  int n_jobs = 0;
  for (int r = 0; r < n_ranks; ++r) {
    size_t b = 0, e = 0;
    ktb_shard_bounds(rows, n_ranks, r, &b, &e);
    if (stage_in[r] && e > b && std::find(jobs, jobs + n_jobs, devs[r]) == jobs + n_jobs) jobs[n_jobs++] = devs[r];
  }
  HostWorker* posted[kMaxDevices] = {nullptr};
  for (int j = 1; j < n_jobs; ++j) {
    const int dev = jobs[j];
    posted[j] = worker_for(dev);
    worker_post(posted[j], [=]() { return run_device(dev); });
  }
  int status = KTB_OK;
  char first_err[512] = "";
  if (n_jobs > 0) {   // the first device's job runs on the calling thread (saves one wake-up)
    status = run_device(jobs[0]);
    if (status != KTB_OK) snprintf(first_err, sizeof(first_err), "%s", last_error_cstr());
  }
  for (int j = 1; j < n_jobs; ++j) {
    int rc = worker_wait(posted[j]);   // always wait for every job: the buffers are borrowed until then
    if (rc != KTB_OK && status == KTB_OK) status = rc;
  }
  if (first_err[0]) set_error("%s", first_err);
  return status;
}

}  // extern "C"
