// ktb_dispatch.cu — multi-GPU data movement of the remote-map path over NVLink 5 / NVSwitch
// (the host-resident PCIe form of the call is ktb_host.cu).
//
// Replaces the reference's fan-out/fan-in:
//   broadcast of the same params to every rank   kt/serving/spmd/spmd_supervisor.py:341,439-455
//   per-rank mp.Queue put / HTTP POST            kt/serving/process_pool.py:125-212,
//                                                kt/serving/remote_worker_pool.py:254-316
//   concatenation of per-rank results            kt/serving/spmd/spmd_supervisor.py:547-570
// On this route the "wire" is peer-mapped HBM: a rank's kernel loads its shard directly from
// the root GPU's arg arena and stores its result directly into the root's result arena, so
// scatter, exec and gather are one kernel per rank and root HBM is read once / written once.
#include "ktb_common.cuh"

#include <algorithm>
#include <mutex>

namespace ktb {


// ---- broadcast: one read, n peer stores ---------------------------------------------------------
constexpr int kBcastMax = 15;
constexpr int kBcastThreads = 256;
constexpr int kBcastUnroll = 2;

struct BcastDsts {
  uint8_t* d[kBcastMax];
  int n;
};

__global__ void __launch_bounds__(kBcastThreads)
    bcast_kernel(const uint8_t* src, const __grid_constant__ BcastDsts dsts, size_t n_bytes) {
  constexpr size_t VB = 32;
  constexpr size_t ROW = (size_t)kBcastThreads * VB;
  constexpr size_t TILE = ROW * kBcastUnroll;
  const size_t n_full = n_bytes / TILE;
  for (size_t t = blockIdx.x; t < n_full; t += gridDim.x) {
    const size_t off = t * TILE + (size_t)threadIdx.x * VB;
    uint32_t w[kBcastUnroll][8];
#pragma unroll
    for (int j = 0; j < kBcastUnroll; ++j) ldg256(src + off + j * ROW, w[j]);
    for (int k = 0; k < dsts.n; ++k) {
#pragma unroll
      for (int j = 0; j < kBcastUnroll; ++j) stg256(dsts.d[k] + off + j * ROW, w[j]);
    }
  }
  if (blockIdx.x == (unsigned)(n_full % gridDim.x)) {
    const size_t base = n_full * TILE;
    const size_t n_vec = (n_bytes - base) / VB;
    for (size_t v = threadIdx.x; v < n_vec; v += kBcastThreads) {
      uint32_t w[8];
      ldg256(src + base + v * VB, w);
      for (int k = 0; k < dsts.n; ++k) stg256(dsts.d[k] + base + v * VB, w);
    }
    const size_t tail = base + n_vec * VB;
    for (size_t e = tail + threadIdx.x; e < n_bytes; e += kBcastThreads) {
      uint8_t b = src[e];
      for (int k = 0; k < dsts.n; ++k) dsts.d[k][e] = b;
    }
  }
}

// Unaligned fallback.
__global__ void __launch_bounds__(256)
    bcast_bytes_kernel(const uint8_t* src, const __grid_constant__ BcastDsts dsts, size_t n_bytes) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_bytes; e += stride) {
    uint8_t b = src[e];
    for (int k = 0; k < dsts.n; ++k) dsts.d[k][e] = b;
  }
}

}  // namespace ktb

using namespace ktb;

extern "C" {

int ktb_broadcast(int root, const void* src, void* const* dsts, int n_dst, size_t nbytes,
                  uintptr_t stream) {
  int rc = require_device(root);
  if (rc) return rc;
  KTB_REQUIRE(n_dst >= 0 && n_dst <= kBcastMax, KTB_ERR_ARG, "ktb_broadcast: n_dst %d out of range [0,%d]",
              n_dst, kBcastMax);
  if (nbytes == 0 || n_dst == 0) return KTB_OK;
  KTB_REQUIRE(src && dsts, KTB_ERR_ARG, "ktb_broadcast: null argument");
  BcastDsts b;
  b.n = 0;
  uintptr_t align = (uintptr_t)src;
  for (int k = 0; k < n_dst; ++k) {
    KTB_REQUIRE(dsts[k], KTB_ERR_ARG, "ktb_broadcast: dsts[%d] is null", k);
    if (dsts[k] == src) continue;  // the root's own copy
    b.d[b.n++] = static_cast<uint8_t*>(dsts[k]);
    align |= (uintptr_t)dsts[k];
  }
  if (b.n == 0) return KTB_OK;
  KTB_GUARD(root);
  const DeviceInfo* di = device_info(root);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if ((align & 31) == 0) {
    size_t tiles = nbytes / ((size_t)kBcastThreads * 32 * kBcastUnroll);
    int grid = (int)std::min<size_t>(std::max<size_t>(tiles, 1), (size_t)di->sm_count * 4);
    bcast_kernel<<<grid, kBcastThreads, 0, st>>>(static_cast<const uint8_t*>(src), b, nbytes);
  } else {
    size_t blocks = (nbytes + 255) / 256;
    int grid = (int)std::min<size_t>(std::max<size_t>(blocks, 1), (size_t)di->sm_count * 8);
    bcast_bytes_kernel<<<grid, 256, 0, st>>>(static_cast<const uint8_t*>(src), b, nbytes);
  }
  KTB_CK(cudaGetLastError());
  return KTB_OK;
}

}  // extern "C"

// Per-THREAD event pool: each host thread owns its events (per device: slot 0 "args ready", slot 1+r "rank r done"), created
// once and reused by every call the thread makes — a call used to pay N+1 cudaEventCreate/Destroy pairs (≈25 µs at
// N = 8).  Reuse is safe: cudaStreamWaitEvent captures the record that is current WHEN THE WAIT IS ENQUEUED, so
// re-recording the event for the next call does not disturb waits enqueued earlier; and because the pool is
// per thread, two host threads on different streams never see each other's records.
struct CallEvents {
  cudaEvent_t make(int device, int slot) {
    struct Pool {
      cudaEvent_t ev[kMaxDevices][kMaxDevices + 1] = {};
      ~Pool() {}   // events die with the context at process exit (destroying them here could outlive the driver)
    };
    static thread_local Pool pool;
    if (device < 0 || device >= kMaxDevices || slot < 0 || slot > kMaxDevices) return nullptr;
    cudaEvent_t& e = pool.ev[device][slot];
    if (!e) {
      DeviceGuard g(device);
      if (!g.ok || cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) {
        e = nullptr;
        return nullptr;
      }
    }
    return e;
  }
};

static int check_ranks(const char* who, int n_ranks, const int* devs, int root_rank) {
  KTB_REQUIRE(n_ranks > 0 && n_ranks <= kMaxDevices && devs, KTB_ERR_ARG, "%s: bad n_ranks %d", who, n_ranks);
  KTB_REQUIRE(root_rank >= 0 && root_rank < n_ranks, KTB_ERR_ARG, "%s: root_rank %d out of range", who, root_rank);
  for (int r = 0; r < n_ranks; ++r) {
    int rc = require_device(devs[r]);
    if (rc) return rc;
    if (devs[r] != devs[root_rank]) {
      KTB_REQUIRE(ktb_peer_enabled(devs[r], devs[root_rank]) == 1, KTB_ERR_UNSUPPORTED,
                  "%s: device %d has no peer access to root device %d", who, devs[r], devs[root_rank]);
    }
  }
  return KTB_OK;
}

// streams == NULL → library streams; otherwise streams[r] verbatim (0 is the legacy default stream)
static cudaStream_t rank_stream(const uintptr_t* streams, const int* devs, int r) {
  return streams ? reinterpret_cast<cudaStream_t>(streams[r]) : device_info(devs[r])->stream_rank;
}

// The fork/join of the scatter forms: record "args ready" on the root stream; per rank, order the rank's stream
// after it, run launch(r, dev, b, e, stream) on elements [b, e) of its shard and record "rank r done"; then join
// every rank on the root stream.  A rank on the root stream itself needs no events.  With skip_empty, a rank whose
// shard is empty is skipped outright (no launch, no events).
template <class Launch>
static int fork_join(const char* who, size_t n_elems, size_t granule, int n_ranks, const int* devs, int root_rank,
                     const uintptr_t* streams, bool skip_empty, Launch&& launch) {
  const int root_dev = devs[root_rank];
  cudaStream_t root_stream = rank_stream(streams, devs, root_rank);
  CallEvents events;
  cudaEvent_t done[kMaxDevices] = {nullptr};
  cudaEvent_t args_ready = events.make(root_dev, 0);
  KTB_REQUIRE(args_ready, KTB_ERR_CUDA, "%s: cudaEventCreate failed", who);
  {
    KTB_GUARD(root_dev);
    KTB_CK(cudaEventRecord(args_ready, root_stream));  // args are ready on the root
  }
  for (int r = 0; r < n_ranks; ++r) {
    size_t b = 0, e = 0;
    ktb_shard_bounds(n_elems / granule, n_ranks, r, &b, &e);
    b *= granule;
    e *= granule;
    if (skip_empty && e == b) continue;
    const int dev = devs[r];
    KTB_GUARD(dev);
    cudaStream_t st = rank_stream(streams, devs, r);
    // same ordering domain as the root only if it is the same stream ON the same device (handle 0 is
    // "the default stream of whichever device is current", so handles alone do not identify a stream)
    const bool is_root = (r == root_rank) || (dev == root_dev && st == root_stream);
    if (!is_root) KTB_CK(cudaStreamWaitEvent(st, args_ready, 0));
    int rc = launch(r, dev, b, e, st);
    if (rc) return rc;
    if (!is_root) {
      done[r] = events.make(dev, 1 + r);
      KTB_REQUIRE(done[r], KTB_ERR_CUDA, "%s: cudaEventCreate failed", who);
      KTB_CK(cudaEventRecord(done[r], st));
    }
  }
  // Join on the root stream with the ROOT device current: stream handle 0 names the default stream of
  // whichever device is current, so the wait must be issued under the root's guard.
  KTB_GUARD(root_dev);
  for (int r = 0; r < n_ranks; ++r)
    if (done[r]) KTB_CK(cudaStreamWaitEvent(root_stream, done[r], 0));
  return KTB_OK;
}

extern "C" {

int ktb_scatter_map_gather(int op, int dtype, const void* src_root, void* dst_root, size_t n_elems,
                           size_t granule, double alpha, double beta, int n_ranks, const int* devs,
                           int root_rank, int variant, const uintptr_t* streams) {
  int rc = check_ranks("ktb_scatter_map_gather", n_ranks, devs, root_rank);
  if (rc) return rc;
  if (n_elems == 0) return check_dtype("ktb_scatter_map_gather", dtype);   // an empty call checks the dtype only
  rc = check_elementwise("ktb_scatter_map_gather", op, dtype);   // before the fork: nothing is queued for a bad op
  if (rc) return rc;
  const size_t es = dtype_size(dtype);
  KTB_REQUIRE(src_root && dst_root, KTB_ERR_ARG, "ktb_scatter_map_gather: null src/dst");
  KTB_REQUIRE(granule > 0 && n_elems % granule == 0, KTB_ERR_ARG,
              "ktb_scatter_map_gather: n_elems %zu is not a multiple of granule %zu", n_elems, granule);
  const MapParams p = make_params(alpha, beta, dtype);
  return fork_join("ktb_scatter_map_gather", n_elems, granule, n_ranks, devs, root_rank, streams, true,
                   [&](int, int dev, size_t b, size_t e, cudaStream_t st) {
                     return launch_map(dev, op, dtype, static_cast<const uint8_t*>(src_root) + b * es,
                                       static_cast<uint8_t*>(dst_root) + b * es, e - b, p, variant, st);
                   });
}

int ktb_scatter_map_reduce(int op, int dtype, const void* src_root, size_t n_elems, size_t granule,
                           double alpha, double beta, int n_ranks, const int* devs, int root_rank,
                           void* partials_root, void* out_root, void* const* workspaces,
                           const uintptr_t* streams) {
  int rc = check_ranks("ktb_scatter_map_reduce", n_ranks, devs, root_rank);
  if (rc) return rc;
  rc = check_reducible("ktb_scatter_map_reduce", op, dtype);
  if (rc) return rc;
  const size_t es = dtype_size(dtype);
  KTB_REQUIRE(partials_root && out_root && workspaces, KTB_ERR_ARG, "ktb_scatter_map_reduce: null argument");
  for (int r = 0; r < n_ranks; ++r)
    KTB_REQUIRE(workspaces[r], KTB_ERR_ARG, "ktb_scatter_map_reduce: workspaces[%d] is null", r);
  KTB_REQUIRE(src_root || n_elems == 0, KTB_ERR_ARG, "ktb_scatter_map_reduce: null src");
  KTB_REQUIRE(granule > 0 && n_elems % granule == 0, KTB_ERR_ARG,
              "ktb_scatter_map_reduce: n_elems %zu is not a multiple of granule %zu", n_elems, granule);
  const MapParams p = make_params(alpha, beta, dtype);
  // empty shards still launch: they write a zero partial (n_elems = 0 → kernel stores 0)
  rc = fork_join("ktb_scatter_map_reduce", n_elems, granule, n_ranks, devs, root_rank, streams, false,
                 [&](int r, int dev, size_t b, size_t e, cudaStream_t st) {
                   return launch_map_reduce(dev, op, dtype, static_cast<const uint8_t*>(src_root) + b * es, e - b, p,
                                            static_cast<uint8_t*>(partials_root) + (size_t)r * acc_size(dtype),
                                            workspaces[r], st);
                 });
  if (rc) return rc;
  KTB_GUARD(devs[root_rank]);
  return launch_reduce_partials(devs[root_rank], dtype, partials_root, n_ranks, out_root,
                                rank_stream(streams, devs, root_rank));
}

// ktb_map_host_multi (host-resident args over PCIe) lives in ktb_host.cu.

}  // extern "C"
